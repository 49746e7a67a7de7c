"""L2 framing on the device (SURVEY §8 f1, nrsc5_b200/csrc/l2.cuh) against the oracle's L2 restatement - which is
pinned, byte for byte, to the unmodified reference's L2 -> L3 calls (tests/test_oracle_l2.py) - and against the
golden call streams made from the reference (tests/golden/l2.json).  Through the C ABI: nrsc5b_l2_frames (L2
alone, all six frame lengths) and nrsc5b_enable_l2 (the whole chain, REC_L2 after every frame's pass).

They went green on the CPU emulation of the kernels first (tests/test_emu_engine.py runs these very functions) and
then on the GPU."""
import os

import pytest

import port
from common import FM_MODE_CASES, MP3_CASE, SYNTH_CASES, golden, load_sample
from l2_cases import L2_CASES, l2_digest, malformed_sequences, mutated_sequence, stress_sequences
from nrsc5_b200 import engine as eng
from nrsc5_b200 import synth, synth_l2

pytestmark = pytest.mark.gpu


def expand(l2_records, frames):
    """REC_L2 records of nrsc5b_l2_frames -> the oracle's flat stream: every frame followed by its calls."""
    pushed = [f for f in frames if f is not None]
    out = []
    for r in l2_records:
        lc, nbits, bits = pushed[r["ordinal"]]
        out.append((1, {"lc": lc, "nbits": nbits, "bits": bytes(bits[:(nbits + 7) // 8])}))
        out.extend(r["events"])
    return out


@pytest.mark.parametrize("name", sorted(L2_CASES))
def test_l2_frames_equal_oracle(name):
    frames = synth_l2.make_l2_sequence(**L2_CASES[name])
    recs = eng.l2_frames(frames)
    orc, lost = port.l2_frames(frames)
    got = expand(recs, frames)
    assert len(recs) == sum(f is not None for f in frames)
    assert got == orc.records                                # same calls, same order, same bytes
    assert l2_digest(got) == golden("l2.json")[name]         # = the unmodified reference
    assert sum(bool(r["flags"] & eng.L2F_LOST) for r in recs) == lost
    assert not any(r["flags"] & eng.L2F_EV_OVERFLOW for r in recs)
    for r, f in zip(recs, [f for f in frames if f is not None]):
        assert (r["lc"], r["nbits"]) == (f[0], f[1]) and len(r["pdu"]) == synth_l2.pdu_len(f[1])


@pytest.mark.parametrize("block", range(3))
def test_l2_frames_mutated_equal_oracle(block):
    """PDUs with random byte errors (tests/l2_cases.py:mutated_sequence; the oracle equals the reference on them,
    tests/test_oracle_l2.py): the device takes the same early returns, finds the same packets and CRC verdicts."""
    for trial in range(8 * block, 8 * block + 8):
        frames, _ = mutated_sequence(trial)
        recs = eng.l2_frames(frames)
        orc, lost = port.l2_frames(frames)
        assert expand(recs, frames) == orc.records, trial
        assert sum(bool(r["flags"] & eng.L2F_LOST) for r in recs) == lost, trial


def test_l2_frames_of_sample_xz():
    """The P1 frames the reference decodes from support/sample.xz (here: the oracle's, equal by test_oracle.py)
    through the device L2: 522 packets, 8 PSD messages, 2 service reports, as the reference."""
    cu8 = load_sample()
    if cu8 is None:
        pytest.skip("sample.xz not present")
    frames = port.l1_to_l2_input(port.decode(cu8).records)
    recs = eng.l2_frames(frames)
    got = expand(recs, frames)
    assert l2_digest(got) == golden("l2.json")["sample_xz"]
    assert [bool(r["flags"] & eng.L2F_LOST) for r in recs] == [True] + [False] * 8


def test_chain_with_l2_on_device():
    """Whole chain with nrsc5b_enable_l2: a capture whose P1 PDUs carry real audio PDUs; the records, with every
    REC_L2 put behind its frame, equal the oracle's L1 stream with the oracle's L2 calls after every frame."""
    frames = [f for f in synth_l2.make_l2_sequence(seed=21, nframes=3) if f is not None]
    # the first L1 frame after acquisition is decoded from blocks the tracking loops were still converging on
    # (channel BER 0.14 in the reference too): it keeps the generator's plain PDU, the L2 content starts with the second
    cap = synth.make_fm_mp1(nframes=4, seed=1234, lead_in=1777, p1_frames=[None] + [f[2] for f in frames])
    cu8 = cap.cu8[:cap.cu8.size & ~3]
    half = (cu8.size // 2) & ~3
    # a third channel with other PDUs (and a carrier offset): the per-stream L2 state must not mix
    frames_c = [f for f in synth_l2.make_l2_sequence(seed=22, nframes=3) if f is not None]
    cap_c = synth.make_fm_mp1(nframes=4, seed=77, lead_in=333, cfo_hz=120.0, p1_frames=[None] + [f[2] for f in frames_c])
    cu8_c = cap_c.cu8[:cap_c.cu8.size & ~3]
    with eng.Engine(nstreams=3, input_capacity=max(cu8.size, cu8_c.size) + 4096, log_capacity=1 << 20) as e:
        e.enable_l2()
        e.push_cu8(0, cu8)
        e.push_cu8(1, cu8[:half])
        e.push_cu8(2, cu8_c)
        e.process()
        e.push_cu8(1, cu8[half:])
        e.process()
        raws = [e.drain_raw(0), e.drain_raw(1), e.drain_raw(2)]
    l1 = port.decode(cu8)
    want = []
    l2in, l2 = port.l1_to_l2_input(l1.records), None
    orc, _ = port.l2_frames(l2in)
    calls = iter(orc.records)
    nxt = next(calls, None)
    for ty, r in l1.records:
        if ty in (eng.REC_SOFT_PM, eng.REC_BLOCK):
            continue
        want.append((ty, r))
        if ty == eng.REC_FRAME:
            assert nxt is not None and nxt[0] == 1
            nxt = next(calls, None)
            while nxt is not None and nxt[0] != 1:
                want.append(nxt)
                nxt = next(calls, None)
    for raw in raws[:1]:
        got = [(t, r) for t, r in eng.with_l2_in_call_order(raw) if t != eng.REC_BLOCK]
        key = lambda t, r: (t, r.get("bits"), r.get("data"), r.get("seq"), r.get("offset"), r.get("program"))
        gk, wk = [key(t, r) for t, r in got], [key(t, r) for t, r in want]
        i0 = next(i for i, k in enumerate(wk) if k[0] == 1)
        gk[i0] = wk[i0] = (1,)                                # that first frame: bits not compared
        assert gk == wk
        assert sum(1 for t, _ in got if t == eng.EV_PACKET) > 50
    # the second stream got its input in two pushes and two passes: same frames, same L2 calls
    a = [(t, r) for t, r in eng.with_l2_in_call_order(raws[0]) if t in (16, 17, 18, 19)]
    b = [(t, r) for t, r in eng.with_l2_in_call_order(raws[1]) if t in (16, 17, 18, 19)]
    assert a == b and len(a) > 50
    # the third channel: its own frames, its own calls
    l1c = [(t, r) for t, r in eng.parse_records(raws[2]) if t in (1, 3)]
    orc_c, _ = port.l2_frames(port.l1_to_l2_input(l1c))
    c = [(t, r) for t, r in eng.with_l2_in_call_order(raws[2]) if t in (1, 16, 17, 18, 19)]
    assert c == orc_c.records and [r for t, r in c if t != 1] != [r for t, r in a]
    assert [r["bits"] for t, r in c if t == 1][1:] == [f[2] for f in frames_c]


def test_mp3_chain_l2_records_follow_their_frames():
    """MP3: P1 and P3 frames of one pass go through L2 in the reference's call order (P3 frames of the odd blocks,
    the P1 frame before the P3 frame of block 15); every REC_FRAME gets exactly one REC_L2 naming it, and the calls
    equal the oracle's L2 over the same L1 stream."""
    cap = synth.make_fm_mp3(**MP3_CASE)
    cu8 = cap.cu8[:cap.cu8.size & ~3]
    with eng.Engine(nstreams=1, input_capacity=cu8.size + 4096, log_capacity=4 << 20) as e:
        e.enable_l2()
        e.push_cu8(0, cu8)
        e.process()
        raw = e.drain_raw(0)
    offs = []
    recs = eng.parse_records(raw, offs)
    frames = {at: r for (t, r), at in zip(recs, offs) if t == eng.REC_FRAME}
    l2s = [r for t, r in recs if t == eng.REC_L2]
    assert len(l2s) == len(frames) >= 20 and {r["frame_rec_off"] for r in l2s} == set(frames)
    for r in l2s:
        f = frames[r["frame_rec_off"]]
        assert (r["lc"], r["nbits"]) == (f["lc"], f["nbits"])
    assert [r["ordinal"] for r in l2s] == list(range(len(l2s)))
    # L2 takes the frames in log order = the reference's call order
    assert [r["frame_rec_off"] for r in l2s] == sorted(frames)
    got = [(t, r) for t, r in eng.with_l2_in_call_order(raw) if t in (1, 16, 17, 18, 19)]
    orc, _ = port.l2_frames(port.l1_to_l2_input([(t, r) for t, r in recs if t in (1, 3)]))
    assert got == orc.records


def test_dropin_with_device_l2_matches_reference_events():
    """The drop-in libnrsc5.so with NRSC5_B200_DEVICE_L2=1 through the reference's public API on sample.xz: the
    seam replays REC_L2 instead of calling frame_push(); same events, 476 identical HDC packets, ID3, AUDIO_SERVICE."""
    import test_dropin
    try:
        test_dropin.test_dropin_events_match_reference_on_sample_xz(1)
    finally:
        os.environ.pop("NRSC5_B200_DEVICE_L2", None)


def test_am_chain_with_l2_on_device():
    """AM (MA1): the 3750-bit P1 frames carry real audio PDUs; with nrsc5b_enable_l2 an AM engine hands every frame
    k_am decodes to k_l2 (launches of at most 16 blocks each), and the records equal the oracle's L1 stream with the
    oracle's L2 calls behind every frame."""
    from nrsc5_b200 import synth_am
    src = [f for f in synth_l2.make_l2_sequence(seed=33, nframes=13 * 8, nbits=3750) if f is not None]
    # frames the generator made uncorrectable on purpose would drop sync in AM (frame.c:538): keep the decodable ones
    good = [f[2] for i, f in enumerate(src) if i % 12 != 5]
    cap = synth_am.make_am_ma1(nframes=10, seed=3, lead_in=500, p1_frames=good)
    with eng.Engine(nstreams=1, input_capacity=4 * cap.cs16.size + 4096, log_capacity=1 << 20, mode="am") as e:
        e.enable_l2()
        e.push_cs16(0, cap.cs16)
        e.process()
        raw = e.drain_raw(0)
    l1 = port.decode_am(cap.cs16)
    orc, lost = port.l2_frames(port.l1_to_l2_input(l1.records))
    got = [(t, r) for t, r in eng.with_l2_in_call_order(raw) if t in (1, 16, 17, 18, 19)]
    assert got == orc.records
    assert sum(1 for t, _ in got if t == 19) > 60 and lost == 0
    assert [t for t, _ in eng.parse_records(raw) if t != eng.REC_L2] == [t for t, _ in l1.records]


@pytest.mark.parametrize("psmi,fmt", [(1, "cs16"), (2, "cu8")])
def test_dropin_am_with_device_l2_matches_reference_events(psmi, fmt):
    """AM through the drop-in's public API with NRSC5_B200_DEVICE_L2=1 (AM frames through k_l2 as well)."""
    import test_dropin
    os.environ["NRSC5_B200_DEVICE_L2"] = "1"
    try:
        test_dropin.test_dropin_am_matches_reference_events(psmi, fmt)
    finally:
        os.environ.pop("NRSC5_B200_DEVICE_L2", None)


@pytest.mark.parametrize("mode", ["mp2", "mp11"])
def test_service_mode_chain_l2_call_order(mode):
    """MP2 (2304-bit P3 frames) and MP11 (P3 and P4 frames, decode groups added to the passes on demand): every
    frame of every logical channel gets its REC_L2, taken in the reference's call order (P1 before the P3 / P4 frames
    of block 15, P3 before P4), and the calls equal the oracle's L2 over the same frames."""
    cap = synth.make_fm(**FM_MODE_CASES[mode])
    cu8 = cap.cu8[:cap.cu8.size & ~3]
    with eng.Engine(nstreams=1, input_capacity=cu8.size + 4096, log_capacity=4 << 20) as e:
        e.enable_l2()
        e.push_cu8(0, cu8)
        e.process()
        raw = e.drain_raw(0)
    offs = []
    recs = eng.parse_records(raw, offs)
    frames = {at: r for (t, r), at in zip(recs, offs) if t == eng.REC_FRAME}
    l2s = [r for t, r in recs if t == eng.REC_L2]
    assert [r["frame_rec_off"] for r in l2s] == sorted(frames) and len(l2s) >= 10
    assert {r["lc"] for r in l2s} == ({0, 1} if mode == "mp2" else {0, 1, 2})
    got = [(t, r) for t, r in eng.with_l2_in_call_order(raw) if t in (1, 16, 17, 18, 19)]
    orc, _ = port.l2_frames(port.l1_to_l2_input([(t, r) for t, r in recs if t in (1, 3)]))
    assert got == orc.records


@pytest.mark.parametrize("name", ["ccc_overlong", "hef_past_la"])
def test_l2_malformed_pdus_stay_in_bounds(name):
    """PDUs on which the reference's frame.c leaves its buffers (tests/l2_cases.py:malformed_sequences): the kernel
    must neither fault nor differ from the oracle's defined outcome, and must carry on with the next frames."""
    frames = malformed_sequences()[name]
    recs = eng.l2_frames(frames)
    orc, _ = port.l2_frames(frames)
    assert expand(recs, frames) == orc.records
    assert len(recs) == len(frames) - 1
    if name == "ccc_overlong":
        assert sum(len(r["events"]) for r in recs[:3]) > 0 and all(not r["events"] for r in recs[-4:])
    else:
        assert all(any(t == eng.EV_PACKET for t, _ in r["events"]) for r in recs)


def test_mp3_chain_with_l2_content_in_p3_frames():
    """MP3 with real audio PDUs in the P3 frames (and plain ones in P1): both logical channels feed the same service
    table and PSD buffers, so the interleaving of the P1 and P3 frames' calls - P3 frames of the odd blocks, the P1
    frame ahead of block 15's P3 frame - shows in the events; they must equal the oracle's L2 over the same frames."""
    src = [f for f in synth_l2.make_l2_sequence(seed=44, nframes=34, nbits=4608, lc=1) if f is not None]
    cap = synth.make_fm_mp3(**MP3_CASE, p3_frames=[f[2] for f in src])
    cu8 = cap.cu8[:cap.cu8.size & ~3]
    with eng.Engine(nstreams=1, input_capacity=cu8.size + 4096, log_capacity=4 << 20) as e:
        e.enable_l2()
        e.push_cu8(0, cu8)
        e.process()
        raw = e.drain_raw(0)
    recs = eng.parse_records(raw)
    got = [(t, r) for t, r in eng.with_l2_in_call_order(raw) if t in (1, 16, 17, 18, 19)]
    orc, _ = port.l2_frames(port.l1_to_l2_input([(t, r) for t, r in recs if t in (1, 3)]))
    assert got == orc.records
    p3 = [r["bits"] for t, r in recs if t == 1 and r["lc"] == 1]
    assert len(p3) >= 12 and all(b in {f[2] for f in src} for b in p3)      # decoded P3 frames = generated ones
    assert sum(1 for t, _ in got if t == 19) > 30 and sum(1 for t, _ in got if t == 16) >= 4


def test_am_rewind_repeats_the_decode():
    """nrsc5b_rewind on an AM engine: the receiver state (AmState / AmWork, and the L2 state) starts over on the
    samples the engine already holds; the second pass writes the same records as the first."""
    from nrsc5_b200 import synth_am
    cap = synth_am.make_am_ma1(nframes=9, seed=3, lead_in=500)
    with eng.Engine(nstreams=2, input_capacity=4 * cap.cs16.size + 4096, log_capacity=1 << 20, mode="am") as e:
        e.enable_l2()
        e.push_cs16(0, cap.cs16)
        e.push_cs16(1, cap.cs16[:cap.cs16.size // 2 & ~1])
        e.process()
        first = [e.drain_raw(0), e.drain_raw(1)]
        e.rewind()
        e.process()
        second = [e.drain_raw(0), e.drain_raw(1)]
    assert first == second and len(first[0]) > len(first[1]) > 0
    assert sum(1 for t, _ in eng.parse_records(first[0]) if t == eng.REC_L2) >= 8


@pytest.mark.parametrize("name", ["many_packets", "hdlc_overrun", "ev_overflow"])
def test_l2_rare_branches(name):
    """More packets per frame (2268) than the kernel's packet table holds (thread 0 checks those CRCs itself), an HDLC
    buffer overrun, and more events than the per-frame staging area holds: the first two equal the oracle (which
    equals the reference on them); the third sets L2F_EV_OVERFLOW and keeps a prefix of the calls."""
    frames = stress_sequences()[name]
    recs = eng.l2_frames(frames)
    orc, _ = port.l2_frames(frames)
    got = expand(recs, frames)
    if name != "ev_overflow":
        assert got == orc.records and not any(r["flags"] & eng.L2F_EV_OVERFLOW for r in recs)
        assert max(sum(1 for t, _ in r["events"] if t == eng.EV_PACKET) for r in recs) >= (2268 if name == "many_packets" else 400)
    else:
        assert recs[0]["flags"] & eng.L2F_EV_OVERFLOW
        assert 2000 < len(got) < len(orc.records) and got == orc.records[:len(got)]
