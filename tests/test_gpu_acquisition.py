"""GPU parity of coarse acquisition and of the integer-CFO search, against the oracle: captures whose search picks an
offset other than its first trial, searches that find nothing, acquisition windows at every word phase, and streams
with less lead-in than one window (the first tiles see the zero fill).

Every block's parameters (REC_BLOCK: state, timing, integer CFO, window start) must equal the oracle's, as must the
PDUs and the order of every call.  Every test runs with one CTA per stream (NRSC5_B200_CLUSTER=1: k_stream<false>,
whose acquisition is front_prep_single) and with the default cluster of a one-stream engine (k_stream<true>,
front_acq_tiles / front_acq_corr).  The CPU twins run on the emulated kernels (tests/test_emu_acquisition.py)."""
import numpy as np
import pytest

import common
import port
import reftap
from nrsc5_b200 import engine as eng
from nrsc5_b200 import synth
from test_gpu_chain import kinds, oracle_kinds, run_engine

pytestmark = pytest.mark.gpu

SUBCARRIER_HZ = 744187.5 / 2048
CLUSTERS = pytest.mark.parametrize("cluster", ["1", None], ids=["one_cta", "default_cluster"])


def set_cluster(monkeypatch, cluster):
    if cluster is None:
        monkeypatch.delenv("NRSC5_B200_CLUSTER", raising=False)
    else:
        monkeypatch.setenv("NRSC5_B200_CLUSTER", cluster)


def word_phase(start):
    """Where an acquisition window's tiles start in a 16-byte piece of the input: the word of the first halfband input
    of its first tile, start - 38, modulo 4."""
    return (start - 38) & 3


def blocks(recs):
    return [(r["state"], r["samperr"], r["cfo"], r["start"]) for t, r in recs if t == eng.REC_BLOCK]


def oracle_blocks(ref):
    return [(r["state"], r["samperr"], r["cfo"], r["start"]) for r in ref.of(reftap.REC_BLOCK)]


def same_as_oracle(cu8):
    """Run one stream through the engine and the oracle; every block, PDU and call must agree.  Returns the blocks."""
    cu8 = cu8[: cu8.size & ~3]
    ref = port.decode(cu8, want_blocks=True)
    recs = run_engine([cu8])[0]
    got = blocks(recs)
    assert got == oracle_blocks(ref)
    assert [r["bits"] for t, r in recs if t == eng.REC_FRAME] == ref.p1_frames
    assert [r["bits"] for t, r in recs if t == eng.REC_PIDS] == ref.pids_frames
    assert kinds(recs) == oracle_kinds(ref)
    syncs = [r for t, r in recs if t == eng.REC_SYNC]
    want = ref.of(reftap.REC_SYNC)
    assert len(syncs) == len(want)
    for a, b in zip(syncs, want):                 # (the fractional part comes from the FFT arithmetic)
        assert a["psmi"] == b["psmi"] and abs(a["freq_offset"] - b["freq_offset"]) < 0.05
    return got


@CLUSTERS
@pytest.mark.parametrize("k", [-3, -1, 1, 3, 5])
def test_cfo_search_winner_off_its_first_trial(k, cluster, monkeypatch):
    """k subcarriers (plus a fraction) off: the search's winner is the correction -k, not its first trial (-38)."""
    set_cluster(monkeypatch, cluster)
    cap = synth.make_fm_mp1(nframes=2, seed=77 + k, lead_in=333, cfo_hz=k * SUBCARRIER_HZ + 40.0)
    got = same_as_oracle(cap.cu8)
    assert -k in {b[2] for b in got}


@CLUSTERS
def test_cfo_search_winner_in_noise(cluster, monkeypatch):
    set_cluster(monkeypatch, cluster)
    cap = synth.make_fm_mp1(**common.SYNTH_CASES["mp1_cfo2000_awgn20"])
    got = same_as_oracle(cap.cu8)
    assert any(b[2] != 0 for b in got)


@CLUSTERS
def test_cfo_search_runs_out(cluster, monkeypatch):
    """Noise first: every block's vote fails and its search finds nothing (no trial has three agreeing carriers).  Then
    a signal 3 subcarriers off: a search wins, and cfo_wait holds off the next searches while the votes settle.  The
    windows over the noise start wherever its arg-max puts them: between them they cover every word phase."""
    set_cluster(monkeypatch, cluster)
    cap = synth.make_fm_mp1(nframes=2, seed=5, lead_in=333, cfo_hz=3 * SUBCARRIER_HZ)
    rng = np.random.default_rng(5)
    noise = np.clip(np.rint(127.5 + rng.normal(0.0, 20.0, 8 * 276480)), 0, 255).astype(np.uint8)
    got = same_as_oracle(np.concatenate([noise, cap.cu8]))
    assert all(b[2] == 0 for b in got[:6]) and all(b[0] != 2 for b in got[:6])
    assert -3 in {b[2] for b in got} and any(b[0] == 2 for b in got)
    assert {word_phase(b[3]) for b in got if b[0] != 2} == {0, 1, 2, 3}


@CLUSTERS
@pytest.mark.parametrize("lead", [0, 4, 41])
def test_acquisition_with_short_lead_in(lead, cluster, monkeypatch):
    """The stream starts `lead` samples before the signal (cut from a capture with a longer lead-in), far less than
    one window: the first window's first tile reaches back before the stream's first sample (the zero fill)."""
    set_cluster(monkeypatch, cluster)
    cap = synth.make_fm_mp1(nframes=2, seed=31 + lead, lead_in=333)
    got = same_as_oracle(cap.cu8[2 * (333 - lead):])
    assert got[0][3] == 0 and word_phase(got[0][3]) == 2     # the first window starts at the stream's first sample
    assert any(b[0] == 2 for b in got)                      # it did reach fine sync
