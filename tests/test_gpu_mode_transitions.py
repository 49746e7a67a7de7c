"""GPU parity when a stream loses sync while P3 / P4 frames are being produced, changes service mode between two
acquisitions, or asks for an extended-partition decode group in the middle of a run - against the oracle, whose
record stream on the same captures equals the unmodified reference's (tests/test_oracle_mode_transitions.py).

The captures are built in tests/mode_transitions.py.  Their CPU twins run on the emulated kernels
(tests/test_emu_engine.py)."""
import pytest

import mode_transitions as mt
import port
import reftap
import nrsc5_b200
from nrsc5_b200 import engine as eng
from test_gpu_am import digest, oracle_digest, run_am
from test_gpu_chain import run_engine

pytestmark = pytest.mark.gpu


def tokens(recs):
    """The calls that carry the order: F<lc>, S<psmi>, L, B (P and M come once per block and are compared apart)."""
    out = []
    for t, r in recs:
        if t == eng.REC_FRAME:
            out.append("F%d" % r["lc"])
        elif t == eng.REC_SYNC:
            out.append("S%d" % r["psmi"])
        elif t == eng.REC_LOST_SYNC:
            out.append("L")
        elif t == eng.REC_BER:
            out.append("B")
    return out


def oracle_tokens(log):
    return tokens([(t, p) for t, p in log.records if t in (reftap.REC_FRAME, reftap.REC_SYNC, reftap.REC_LOST_SYNC,
                                                           reftap.REC_BER)])


def all_kinds(recs):
    m = {eng.REC_FRAME: "F", eng.REC_PIDS: "P", eng.REC_SYNC: "S", eng.REC_LOST_SYNC: "L", eng.REC_MER: "M", eng.REC_BER: "B"}
    return [m[t] for t, _ in recs if t in m]


def loss_windows(toks, after):
    """What surrounds every sync loss: the two calls before it and `after` calls behind it."""
    return [toks[i - 2: i + 1 + after] for i, x in enumerate(toks) if x == "L"]


def same_as_oracle(recs, ref, exact=None):
    """Frames (lc, nbits, bits), PIDS, every call in order and the service mode of every acquisition equal the
    oracle's.  exact: compare the bits only of frames / PIDS the oracle decoded to one of these (transmitted) PDUs,
    the others by (lc, nbits) / presence; returns how many frames were compared bit for bit."""
    got = [(r["lc"], r["nbits"], r["bits"]) for t, r in recs if t == eng.REC_FRAME]
    want = [(p["lc"], p["nbits"], p["bits"]) for t, p in ref.records if t == reftap.REC_FRAME]
    gp = [r["bits"] for t, r in recs if t == eng.REC_PIDS]
    wp = ref.pids_frames
    assert [f[:2] for f in got] == [f[:2] for f in want]
    if exact is None:
        assert got == want
        assert gp == wp
        n = len(got)
    else:
        frames, pids = exact
        both = [(a, b) for a, b in zip(got, want) if b[2] in frames]
        assert [a for a, _ in both] == [b for _, b in both]
        assert [a for a, b in zip(gp, wp) if b in pids] == [b for b in wp if b in pids]
        n = len(both)
    assert all_kinds(recs) == [e for e in all_kinds(ref.records)]
    assert tokens(recs) == oracle_tokens(ref)
    return n


def run_async(caps, piece=1 << 20, input_capacity=6 << 20):
    """stage / submit / poll (the path the drop-in runs on), one batch in flight, into a buffer far smaller than the
    captures: the records of every batch, concatenated."""
    caps = [c[: c.size & ~3] for c in caps]
    got = [[] for _ in caps]
    with nrsc5_b200.Engine(nstreams=len(caps), input_capacity=input_capacity, log_capacity=8 << 20) as e:
        def take():
            for s in range(len(caps)):
                got[s] += e.batch_records(s)
        waits = 0
        for off in range(0, max(c.size for c in caps), piece):
            for s, c in enumerate(caps):
                p = c[off: off + piece]
                if not p.size:
                    continue
                rc = e.stage_cu8(s, p)
                while rc == -5:
                    waits += 1
                    assert waits < 100000, "the engine never made room"
                    if e.poll(True) == 1:
                        take()
                    e.submit()
                    rc = e.stage_cu8(s, b"")
            if e.poll(False) == 1:
                take()
            e.submit()
        while True:
            if e.poll(True) == 1:
                take()
            if e.submit(True) != 1:
                break
    return [[(t, r) for t, r in g if t != eng.REC_BLOCK] for g in got]


@pytest.mark.parametrize("name", list(mt.LOSS_CASES))
def test_sync_loss_while_px_frames_flow(name):
    """The P1 frame of block 15 fails its header check in MP3, MP11 and MP2 while P3 (and P4) frames come out.  The
    reference reports the loss inside frame_push, i.e. inside decode_push_pm, before decode_push_px1 / _px2 hand
    over that block's P3 / P4 frames: B F0 L F1 [F2]."""
    cu8 = mt.cu8_of([mt.loss_capture(name)])
    ref = port.decode(cu8)
    recs = run_engine([cu8])[0]
    same_as_oracle(recs, ref)
    px = ["F1", "F2"] if name == "mp11" else ["F1"]
    assert loss_windows(tokens(recs), len(px)) == [["B", "F0", "L"] + px]
    assert tokens(recs).count("F1") >= 10


def _check_chain(recs, ref, exact=None):
    n = same_as_oracle(recs, ref, exact)
    syncs = [r["psmi"] for t, r in recs if t == eng.REC_SYNC]
    assert syncs == [p["psmi"] for p in ref.of(reftap.REC_SYNC)]
    assert {1, 2, 3, 11} <= set(syncs)                       # every link was acquired in its own mode
    return n


@pytest.mark.parametrize("how", ["oneshot", "chunked", "async"])
def test_mode_chain_in_one_stream(how):
    """One stream through MP11 -> MP1 -> MP3 -> MP2 -> MP11, every link ending in a P1 frame that loses sync.  After a
    loss the coarse vote still counts the old mode's partitions (sync.c:343-386: psmi survives the loss), the PX1
    ring is reused with another frame length (MP3 -> MP2), P3 / P4 stop (MP11 -> MP1).  The receiver may lock back
    onto the tail of a link and lose sync again on the frame across the seam; all of it must come out as in the
    oracle, whether pushed at once, in pieces that split blocks, or through the asynchronous path.
    A P1 frame decoded across a seam is no codeword (its blocks come from two transmissions); on such a frame
    soft bits that differ from the oracle's by one step (test_gpu_modes.py) can move the Viterbi decision - in
    this chain 1 of 101 frames, the one across the MP2 -> MP11 seam, in the CPU emulation of the kernels, the same
    one-shot and asynchronous.  So frames compare as in test_mode_chain_across_dropouts: bit for bit when the
    oracle decoded a transmitted PDU, by (lc, nbits) otherwise - at most one per seam."""
    links = mt.chain_links()
    cu8 = mt.cu8_of(links)
    ref = port.decode(cu8)
    if how == "oneshot":
        recs = run_engine([cu8])[0]
    elif how == "chunked":
        recs = run_engine([cu8], chunk=3 << 20)[0]           # 11.4 blocks per push
    else:
        recs = run_async([cu8])[0]
    n = _check_chain(recs, ref, exact=mt.transmitted(links))
    assert n >= sum(1 for t, _ in recs if t == eng.REC_FRAME) - (len(links) - 1)
    wins = loss_windows(tokens(recs), 2)
    assert ["B", "F0", "L", "F1", "F2"] in wins and ["B", "F0", "L", "F1", "S3"] in wins
    assert ["B", "F0", "L", "F1", "S2"] in wins


@pytest.mark.parametrize("cluster", ["1", None])
def test_decode_groups_enabled_mid_run(cluster, monkeypatch):
    """Three streams in one engine, pushed in pieces: MP1 throughout; MP1 -> MP11, so that the P3 and P4 decode
    groups are enabled in the middle of the run; MP3 -> MP1, whose PX1 state must stop producing frames.  Every
    stream equals its own oracle decode, with one CTA per stream and with the default cluster size.
    Frames compare as in test_mode_chain_across_dropouts: the P1 frame decoded across the MP1 -> MP11 seam is
    no codeword (its blocks come from two transmissions), and there 17 of its 146 176 bits come out other than
    in the oracle while every soft bit of the stream is within one step of the oracle's."""
    if cluster is None:
        monkeypatch.delenv("NRSC5_B200_CLUSTER", raising=False)
    else:
        monkeypatch.setenv("NRSC5_B200_CLUSTER", cluster)
    caps, sent = mt.lazy_streams()
    outs = run_engine(caps, chunk=3 << 20)
    for cu8, recs, tx in zip(caps, outs, sent):
        n = same_as_oracle(recs, port.decode(cu8), exact=tx)
        assert n >= sum(1 for t, _ in recs if t == eng.REC_FRAME) - 1
    t0, t1, t2 = (tokens(r) for r in outs)
    assert "L" not in t0 and "F1" not in t0
    assert "S11" in t1 and "F2" in t1[t1.index("S11"):] and "F1" not in t1[:t1.index("S11")]
    assert "F1" in t2 and "S1" in t2 and "F1" not in t2[t2.index("S1"):]


def test_sync_loss_with_l2_on_device():
    """(MP11, as test_sync_loss_while_px_frames_flow) with L2 framing on the device: every frame gets one REC_L2, in
    log order; the sync-loss flag is on the P1 frame's REC_L2 only; the L1 records and the L2 calls equal the
    oracle's."""
    cu8 = mt.cu8_of([mt.loss_capture("mp11")])
    ref = port.decode(cu8)
    with eng.Engine(nstreams=1, input_capacity=cu8.size + 4096, log_capacity=8 << 20) as e:
        e.enable_l2()
        e.push_cu8(0, cu8)
        e.process()
        raw = e.drain_raw(0)
    offs = []
    recs = eng.parse_records(raw, offs)
    same_as_oracle([(t, r) for t, r in recs if t != eng.REC_L2], ref)
    frames = {at: r for (t, r), at in zip(recs, offs) if t == eng.REC_FRAME}
    l2s = [r for t, r in recs if t == eng.REC_L2]
    assert [r["frame_rec_off"] for r in l2s] == sorted(frames)
    lost_at, = [at for (t, _), at in zip(recs, offs) if t == eng.REC_LOST_SYNC]
    p1_before = max(at for at, r in frames.items() if r["lc"] == 0 and at < lost_at)
    assert [r["frame_rec_off"] for r in l2s if r["flags"] & eng.L2F_LOST] == [p1_before]
    got = [(t, r) for t, r in eng.with_l2_in_call_order(raw) if t in (1, 16, 17, 18, 19)]
    orc, lost = port.l2_frames(port.l1_to_l2_input([(t, r) for t, r in recs if t in (1, 3)]))
    assert got == orc.records and lost == 1


@pytest.mark.parametrize("how", ["oneshot", "chunked", "async"])
def test_mode_chain_across_dropouts(how):
    """The chain of test_mode_chain_in_one_stream with valid headers, the links separated by 0.4 s of noise.  The
    order of every call and the service mode of every acquisition compare exactly.  Frames compare bit for bit when
    the oracle decoded a transmitted PDU, i.e. when the frame's interleaver span lies in signal; a frame decoded
    (partly) from the noise may differ in its bits - the soft bits of the fp32 demodulator may differ from the
    reference's by one step, which over noise can move the Viterbi decision - so it compares by (lc, nbits)."""
    links = mt.chain_links(gaps=True)
    cu8 = mt.cu8_of(links)
    ref = port.decode(cu8)
    if how == "oneshot":
        recs = run_engine([cu8])[0]
    elif how == "chunked":
        recs = run_engine([cu8], chunk=3 << 20)[0]
    else:
        recs = run_async([cu8])[0]
    n = _check_chain(recs, ref, exact=mt.transmitted(links))
    assert n >= 0.7 * sum(1 for t, _ in recs if t == eng.REC_FRAME)          # 96 of 128
    assert ["B", "F0", "L", "F1", "F2"] in loss_windows(tokens(recs), 2)


def test_am_mode_changes_after_sync_loss():
    """One AM stream MA1 -> MA3 -> MA1, the first two links ending in a P1 frame that loses sync.  The service mode
    is only re-read in COARSE state (sync.c:649-666) and the old one still steers the PIDS combining
    (sync.c:624-633); whole and in pieces, every record equals the oracle's."""
    x = mt.am_chain()
    want = oracle_digest(port.decode_am(x))
    assert digest(run_am([x])[0]) == want
    assert digest(run_am([x], chunk=(1 << 15) + 2)[0]) == want
    assert sum(1 for e in want if e[0] == "L") >= 2
    syncs = [e[1] for e in want if e[0] == "S"]
    assert 2 in syncs and syncs[0] == syncs[-1] == 1


@pytest.mark.parametrize("psmi", [1, 2])
def test_am_rdbi_set(psmi):
    """rdbi = 1 (reference decode.c:494,523): no P3 frames, the BER over P1 only, MA1's PIDS1 zeroed."""
    x = mt.am_rdbi(psmi)
    want = oracle_digest(port.decode_am(x))
    assert digest(run_am([x])[0]) == want
    assert not any(e[0] == "F" and e[1] == 1 for e in want)
    assert sum(1 for e in want if e[0] == "F") >= 24 and all(e[2][3] == 1 for e in want if e[0] == "S")


@pytest.mark.parametrize("psmi", mt.ALIASES)
def test_psmi_aliases(psmi):
    """PSMI values that compatibility_mode maps onto MP1, MP2 and MP5: decoded as their mode, the raw value in SYNC."""
    cu8 = mt.alias_capture(psmi)
    ref = port.decode(cu8)
    recs = run_engine([cu8])[0]
    same_as_oracle(recs, ref)
    syncs = [r["psmi"] for t, r in recs if t == eng.REC_SYNC]
    assert syncs and set(syncs) == {psmi}


def test_psmi_beyond_the_vote_never_acquires():
    """A PSMI of 16 or more is outside the coarse vote (sync.c:396): neither the engine nor the oracle acquires."""
    cu8 = mt.alias_capture(mt.NEVER)
    assert port.decode(cu8).records == []
    recs = run_engine([cu8])[0]
    assert [t for t, _ in recs if t != eng.REC_BLOCK] == []
