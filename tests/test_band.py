"""The band receiver (include/nrsc5_b200.h: nrsc5b_band_*, csrc/band.cu, nrsc5_b200/band.py).  CPU tier: argument checks
without a device, and the policy's restatement (tests/band_policy.py) on hand-built verdicts.  GPU tier: against the
existing pieces - y, the output of a Channelizer of the same plan pushed the whole capture; every window's rows equal
a Scanner given y[:, wW:(w+1)W] and its flags the restated policy; every session's records equal an Engine given
y[k][n0:n1]; stations that come and go, leakage, ragged pushes from host and device in cu8 and cs16, the AM plan, a
rate stage, a full slot table and windows larger than an engine stream's buffer."""
import ctypes
import math

import numpy as np
import pytest

import band_policy as bp
from nrsc5_b200 import band as bd
from nrsc5_b200.engine import EngineError

EINVAL, ENODEV = -2, -1


def _rows(*triples):
    return [dict(detected=bool(d), score=float(s), timing=int(t)) for d, s, t in triples]


N = (0, 0.0, 0)


# ---------------------------------------------------------------- CPU tier

def test_create_needs_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    cfg, keep = bd.make_config("fm", decim=16, offsets=[-3, 0, 4])
    h = ctypes.c_void_p()
    assert bd._lib().nrsc5b_band_create(ctypes.byref(h), ctypes.byref(cfg)) == ENODEV
    with pytest.raises(EngineError, match="ENODEV"):
        bd.BandReceiver()


@pytest.mark.parametrize("kw", [
    dict(decim=4), dict(decim=12), dict(band="am", decim=16), dict(rate=1000), dict(rate=10000001, decim=16),
    dict(decim=8, offsets=[30]), dict(offsets=[-118]), dict(band="am", offsets=[75]), dict(rate=10000000, decim=16, offsets=[44]),
    dict(offsets=[3, 3]), dict(window_symbols=31), dict(window_symbols=513), dict(hold_windows=0), dict(max_stations=0),
    dict(device=-1),
])
def test_bad_configs_are_refused_before_the_device(kw):
    L = bd._lib()
    cfg, keep = bd.make_config(**kw)
    h = ctypes.c_void_p()
    assert L.nrsc5b_band_create(ctypes.byref(h), ctypes.byref(cfg)) == EINVAL


def test_other_refusals():
    L = bd._lib()
    h = ctypes.c_void_p()
    assert L.nrsc5b_band_create(None, None) == EINVAL
    assert L.nrsc5b_band_create(ctypes.byref(h), None) == EINVAL
    cfg, keep = bd.make_config(offsets=[1])
    cfg.nch = 0                                          # offsets without a count
    assert L.nrsc5b_band_create(ctypes.byref(h), ctypes.byref(cfg)) == EINVAL
    cfg, _ = bd.make_config()
    cfg.nch = 3                                          # a count without offsets
    assert L.nrsc5b_band_create(ctypes.byref(h), ctypes.byref(cfg)) == EINVAL
    assert L.nrsc5b_band_push(None, None, 0) == EINVAL
    assert L.nrsc5b_band_flush(None) == EINVAL
    assert L.nrsc5b_band_windows(None, None, None, None, 0, None) == EINVAL
    assert L.nrsc5b_band_sessions(None, None, 0, None) == EINVAL
    assert L.nrsc5b_band_records(None, 0, None, 0, None) == EINVAL


def test_policy_attach_hold_and_reopen():
    W = 1000
    st = (1, 5.0, 100)
    seq = [[N, N], [st, N], [st, N], [N, N], [st, N], [N, N], [N, N], [N, N], [st, N]]
    flags, sess = bp.run([0, 5], "fm", [_rows(*r) for r in seq], W, hold=2, max_stations=4, end=9500)
    assert [f[0] for f in flags] == [0, 5, 5, 4, 5, 4, 0, 0, 5]
    assert sess == [dict(id=0, channel=0, offset=0, slot=-1, n0=1000, n1=6000, window=1),
                    dict(id=1, channel=0, offset=0, slot=-1, n0=8000, n1=9500, window=8)]


def test_policy_suppression_and_ties():
    W = 10
    # a strong station at m = 0 detected beside itself at m = -1 and m = +1 with its timing
    flags, sess = bp.run([-1, 0, 1], "fm", [_rows((1, 2.0, 50), (1, 9.0, 52), (1, 1.0, 45))], W, 1, 8)
    assert flags[0] == [3, 5, 3] and [s["channel"] for s in sess] == [1]
    # a tie: the smaller offset wins
    flags, sess = bp.run([3, 4], "fm", [_rows((1, 4.0, 7), (1, 4.0, 7))], W, 1, 8)
    assert flags[0] == [5, 3] and [s["offset"] for s in sess] == [3]
    # two grid steps apart (FM): both stations, whatever their timing and scores
    flags, sess = bp.run([3, 5], "fm", [_rows((1, 4.0, 7), (1, 9.0, 7))], W, 1, 8)
    assert flags[0] == [5, 5] and len(sess) == 2
    # AM: two steps is still a neighbour, three is not
    flags, _ = bp.run([0, 2, 5], "am", [_rows((1, 9.0, 100), (1, 1.0, 102), (1, 1.0, 100))], W, 1, 8)
    assert flags[0] == [5, 3, 5]
    # a different timing is another station, even next door; a weaker neighbour that is not detected is nothing
    flags, _ = bp.run([0, 1, 2], "fm", [_rows((1, 9.0, 100), (1, 1.0, 157), N)], W, 1, 8)
    assert flags[0] == [5, 5, 0]


def test_policy_timing_wraps_mod_s():
    W = 10
    for band, S, tol in (("fm", 2160, 56), ("am", 270, 7)):
        flags, _ = bp.run([0, 1], band, [_rows((1, 9.0, S - 3), (1, 1.0, tol - 3))], W, 1, 8)
        assert flags[0] == [5, 3], band                  # tol apart across the wrap: leakage
        flags, _ = bp.run([0, 1], band, [_rows((1, 9.0, S - 3), (1, 1.0, tol - 2))], W, 1, 8)
        assert flags[0] == [5, 5], band                  # one more: a station


def test_policy_full_slot_table():
    W = 100
    a, b, c = (1, 3.0, 10), (1, 3.0, 500), (1, 3.0, 900)
    seq = [[a, b, c], [a, b, c], [N, b, c], [N, b, c], [a, b, N]]
    flags, sess = bp.run([-10, 0, 10], "fm", [_rows(*r) for r in seq], W, hold=2, max_stations=2)
    assert flags[0] == [5, 5, 1 | bp.NO_SLOT] and flags[1] == [5, 5, 9]
    assert flags[2] == [4, 5, 9]                          # a: absent once, still held; c still waits
    assert flags[3] == [0, 5, 5]                          # a closes and c takes its stream in the same window
    assert flags[4] == [9, 5, 4]
    assert [(s["channel"], s["slot"], s["n0"], s["n1"]) for s in sess] == [(0, -1, 0, 300), (1, 1, 0, -1), (2, 0, 300, -1)]


# ---------------------------------------------------------------- GPU tier

def _without_positions(recs):
    """REC_BLOCK carries the block's start in the stream's input buffer, which a trim moves; everything else agrees."""
    from nrsc5_b200 import engine as eng
    return [(t, {k: v for k, v in r.items() if not (t == eng.REC_BLOCK and k == "start")}) for t, r in recs]


def _channel_output(x, offsets, band, decim, rate=None, cu8=False):
    """y: the plan's channels of the whole capture through a Channelizer's streaming push, on the device [nch][2 n]."""
    import torch
    from nrsc5_b200 import channelizer as ch
    with ch.Channelizer(offsets, input_cs16=not cu8, band=band, decim=decim, rate=rate) as c:
        n = ch.stream_outputs(0, x.size, band, decim, rate)
        y = torch.empty((len(offsets), 2 * n), dtype=torch.int16, device="cuda")
        assert c.push_device(x.ctypes.data, x.size, y.data_ptr(), 2 * n) == n
        torch.cuda.synchronize()
    return y


def _receive(x, pieces=None, **kw):
    """The capture through a BandReceiver (in pieces: a list of (a, b) slices of x, numpy or a CUDA tensor); returns its
    windows, sessions and every session's records (raw bytes), taken after the flush."""
    with bd.BandReceiver(**kw) as r:
        for a, b in (pieces or [(0, len(x))]):
            r.push(x[a:b])
        r.flush()
        wins, sess = r.windows(), r.sessions()
        recs = [r.records_raw(s["id"]) for s in sess]
        assert all(r.records_raw(s["id"]) == b"" for s in sess)
        offsets = r.offsets
    return offsets, wins, sess, recs


def _check_verdicts(y, offsets, band, wins, sess, W, hold, max_stations):
    from nrsc5_b200 import scan
    n = y.shape[1] // 2
    assert [w["index"] for w in wins] == list(range(n // W))
    with scan.Scanner(len(offsets), band) as s:
        for w in wins:
            s.push_device(y.data_ptr() + 4 * w["index"] * W, y.shape[1], W)
            assert w["rows"] == s.result(), w["index"]
            s.reset()
    flags, want = bp.run(offsets, band, [w["rows"] for w in wins], W, hold, max_stations, end=n)
    assert [list(w["flags"]) for w in wins] == flags
    assert [{k: v for k, v in s.items() if k != "verdict"} for s in sess] == want
    for s in sess:
        assert s["verdict"] == wins[s["window"]]["rows"][s["channel"]]


def _check_records(y, sess, recs, band, l2=False):
    import nrsc5_b200
    from nrsc5_b200 import engine as eng
    for s, raw in zip(sess, recs):
        part = y[s["channel"], 2 * s["n0"]: 2 * s["n1"]].cpu().numpy()
        with nrsc5_b200.Engine(nstreams=1, input_capacity=2 * part.size + 4096, log_capacity=16 << 20, input_cs16=True,
                               mode=band) as e:
            if l2:
                e.enable_l2()
            e.push_cs16(0, part)
            e.process()
            want = e.drain(0)
        got = eng.parse_records(raw)
        assert _without_positions(got) == _without_positions(want), s


# ---- an FM band at D = 8 (5.9535 MS/s) where stations come and go

D8 = 8
FS8 = D8 * 744187.5
SECONDS = 4.2
# (offset, psmi, rms in cu8 LSB, seed, on at, off at (s))
COMINGS = [(-12, 1, 20.0, 71, 0.0, None),           # A: MP1, present throughout
           (5, 3, 20.0 / 31.6, 72, 1.0, None),      # B: MP3, 30 dB under A, switched on at 1 s
           (17, 11, 8.0, 73, 0.0, 2.5)]             # C: MP11, switched off at 2.5 s
CARRIER8, ANALOG8, SPUR8 = -22, 25, 0


def _place(t, m, fs):
    import torch
    ph = torch.remainder(t * (m * 100e3 / fs), 1.0) * (2 * math.pi)
    return torch.complex(torch.cos(ph), torch.sin(ph))


def _comings_capture():
    """COMINGS plus a carrier, an analogue FM host and a spur in a channel's sideband, as a cu8 capture at 5.9535 MS/s."""
    import torch
    from nrsc5_b200 import synth
    dev = "cuda"
    n = int(SECONDS * 1488375)
    up = D8 // 2
    N = n * up
    t = torch.arange(N, dtype=torch.float64, device=dev)
    wide = torch.zeros(N, dtype=torch.complex128, device=dev)
    caps = []
    for m, psmi, rms, seed, on, off in COMINGS:
        cap = synth.make_fm(psmi=psmi, nframes=3, seed=seed, lead_in=700, tail_blocks=2)
        caps.append(cap)
        raw = np.zeros(2 * n)
        k = min(cap.cu8.size, 2 * n)
        raw[:k] = cap.cu8[:k].astype(np.float64) - 127.0
        x = torch.from_numpy(raw).to(dev).view(-1, 2)
        X = torch.fft.fft(torch.complex(x[:, 0].contiguous(), x[:, 1].contiguous()))
        Y = torch.zeros(N, dtype=torch.complex128, device=dev)
        Y[: n // 2] = X[: n // 2]
        Y[-(n - n // 2):] = X[n // 2:]
        z = torch.fft.ifft(Y) * (up * rms / 20.0)
        if on:
            z = torch.roll(z, int(on * FS8))             # the station starts at `on`
            z[: int(on * FS8)] = 0
        if off:
            z[int(off * FS8):] = 0
        wide += z * _place(t, m, FS8)
        del X, Y, z
    wide += 6.0 * _place(t, CARRIER8, FS8)
    phi = 2 * math.pi * 75e3 / 1e3 * torch.sin(2 * math.pi * 1e3 * t / FS8)
    wide += 6.0 * torch.complex(torch.cos(phi), torch.sin(phi)) * _place(t, ANALOG8, FS8)
    wide += 4.0 * torch.exp(2j * math.pi * 160e3 / FS8 * t) * _place(t, SPUR8, FS8)
    g = torch.Generator(device=dev)
    g.manual_seed(8)
    iq = torch.stack([wide.real, wide.imag], -1) + torch.randn((N, 2), generator=g, device=dev, dtype=torch.float64) * 0.3
    x8 = torch.clamp(torch.round(iq + 127.0), 0, 255).to(torch.uint8).reshape(-1)
    return x8.cpu().numpy(), caps


W8 = 128 * 2160
HOLD = 2


@pytest.fixture(scope="module")
def comings():
    x8, caps = _comings_capture()
    kw = dict(band="fm", decim=D8, window_symbols=128, hold_windows=HOLD, max_stations=8)
    offsets, wins, sess, recs = _receive(x8, **kw)
    y = _channel_output(x8, offsets, "fm", D8, cu8=True)
    return x8, caps, kw, offsets, wins, sess, recs, y


@pytest.mark.gpu
def test_verdicts_equal_the_scan_of_each_window(comings):
    x8, caps, kw, offsets, wins, sess, recs, y = comings
    assert offsets == list(range(-29, 30))
    _check_verdicts(y, offsets, "fm", wins, sess, W8, HOLD, 8)


@pytest.mark.gpu
def test_records_equal_an_engine_given_the_session(comings):
    x8, caps, kw, offsets, wins, sess, recs, y = comings
    _check_records(y, sess, recs, "fm")


@pytest.mark.gpu
def test_records_with_l2_equal_an_engine_given_the_session(comings):
    x8, caps, kw, offsets, wins, sess, recs, y = comings
    _, wins2, sess2, recs2 = _receive(x8, **kw, l2=True)
    assert sess2 == sess and all(np.array_equal(a["flags"], b["flags"]) for a, b in zip(wins, wins2))
    from nrsc5_b200 import engine as eng
    assert any(t == eng.REC_L2 for r in recs2 for t, _ in eng.parse_records(r))
    _check_records(y, sess2, recs2, "fm", l2=True)


@pytest.mark.gpu
def test_stations_come_and_go(comings):
    from nrsc5_b200 import engine as eng, synth
    x8, caps, kw, offsets, wins, sess, recs, y = comings
    assert [s["offset"] for s in sess] == [-12, 17, 5], [(s["offset"], s["n0"], s["n1"]) for s in sess]
    a, c, b = sess
    assert a["n0"] == 0 and a["n1"] == y.shape[1] // 2
    on = 1.0 * 744187.5
    kb = offsets.index(5)
    first = min(w["index"] for w in wins if w["rows"][kb]["detected"])
    assert b["window"] == first and (first + 1) * W8 > on, (first, on / W8)
    assert b["n0"] <= on + 2 * W8
    off = 2.5 * 744187.5
    # silent from the window after the one it goes off in; closed hold_windows windows later
    assert off < c["n1"] <= (int(off // W8) + 1 + HOLD) * W8 and c["n1"] % W8 == 0
    for s, cap in ((a, caps[0]), (b, caps[1])):
        got = eng.parse_records(recs[s["id"]])
        assert any(t == eng.REC_SYNC for t, _ in got), s["offset"]
        p1 = [r["bits"] for t, r in got if t == eng.REC_FRAME and r["lc"] == 0]
        assert p1 and any(synth.pack_bits(f) in p1 for f in cap.p1_frames), s["offset"]


@pytest.mark.gpu
def test_ragged_pushes_from_host_and_device_cu8_and_cs16(comings):
    import torch
    x8, caps, kw, offsets, wins, sess, recs, y = comings
    rng = np.random.default_rng(5)
    cuts, pos = [0], 0
    while pos < x8.size:
        pos = min(x8.size, pos + 2 * int(rng.choice([1, 7, 255, 4099, 60000, 700001])))
        cuts.append(pos)
    pieces = list(zip(cuts[:-1], cuts[1:]))
    x16 = (64 * (x8.astype(np.int16) - 127)).astype(np.int16)
    for data, cs16 in ((x8, False), (torch.from_numpy(x16).cuda(), True), (torch.from_numpy(x8).cuda(), False)):
        _, w2, s2, r2 = _receive(data, pieces, **kw, input_cs16=cs16)
        assert [w["index"] for w in w2] == [w["index"] for w in wins]
        assert all(a["rows"] == b["rows"] and np.array_equal(a["flags"], b["flags"]) for a, b in zip(wins, w2))
        assert s2 == sess and r2 == recs, cs16
    # one page-locked buffer, refilled as soon as each push returns (a live SDR's ring): the push must have read it
    ring = torch.empty(max(b - a for a, b in pieces), dtype=torch.uint8).pin_memory()
    with bd.BandReceiver(**kw) as r:
        for a, b in pieces:
            ring[: b - a].copy_(torch.from_numpy(x8[a:b]))
            r.push((ring.data_ptr(), b - a))
            ring.fill_(0)
        r.flush()
        w2, s2 = r.windows(), r.sessions()
        r2 = [r.records_raw(s["id"]) for s in s2]
    assert all(a["rows"] == b["rows"] for a, b in zip(wins, w2)) and s2 == sess and r2 == recs


@pytest.mark.gpu
def test_windows_larger_than_an_engine_stream_lose_no_sample(comings):
    """512 symbols of FM are 4.4 MB of cs16, more than an engine stream's 4 MiB buffer: each window goes in in pieces,
    the engine running between them."""
    x8, caps, kw, offsets, wins, sess, recs, y = comings
    assert 4 * 512 * 2160 > 4 << 20
    k2 = dict(kw, window_symbols=512, hold_windows=1)
    _, w2, s2, r2 = _receive(x8, **k2)
    _check_verdicts(y, offsets, "fm", w2, s2, 512 * 2160, 1, 8)
    assert {s["offset"] for s in s2} >= {-12, 17}
    _check_records(y, s2, r2, "fm")


# ---- leakage of a station some 60 dB over the noise

@pytest.mark.gpu
@pytest.mark.parametrize("psmi,seed,decim,ws", [(3, 34, 32, 512), (11, 36, 8, 256)])
def test_a_strong_station_is_one_session(psmi, seed, decim, ws):
    """Where the scan detects the station in the channels beside it too, those are flagged as leakage: one session."""
    import torch
    from nrsc5_b200 import synth
    fs, up, n = decim * 744187.5, decim // 2, int(2.2 * 1488375)
    cap = synth.make_fm(psmi=psmi, nframes=2, seed=seed, lead_in=900, tail_blocks=0)
    x = torch.from_numpy(cap.cu8[: 2 * n].astype(np.float64) - 127.0).cuda().view(-1, 2)
    X = torch.fft.fft(torch.complex(x[:, 0].contiguous(), x[:, 1].contiguous()))
    N = up * n
    Y = torch.zeros(N, dtype=torch.complex128, device="cuda")
    Y[: n // 2] = X[: n // 2]
    Y[-(n - n // 2):] = X[n // 2:]
    del X
    t = torch.arange(N, dtype=torch.float64, device="cuda")
    m = 7
    wide = torch.fft.ifft(Y) * (up * 60.0) * _place(t, m, fs)
    del Y, t
    g = torch.Generator(device="cuda")
    g.manual_seed(2)
    sig = float(torch.mean(torch.abs(wide) ** 2))
    sigma = math.sqrt(sig / 1e6 * (fs / 400e3) / 2)                      # 60 dB over the noise in the channel's 400 kHz
    iq = torch.stack([wide.real, wide.imag], -1) + torch.randn((N, 2), generator=g, device="cuda", dtype=torch.float64) * sigma
    del wide
    x16 = torch.clamp(torch.round(iq), -32768, 32767).to(torch.int16).reshape(-1).cpu().numpy()
    offs = list(range(m - 3, m + 4))
    offsets, wins, sess, recs = _receive(x16, band="fm", decim=decim, input_cs16=True, offsets=offs, window_symbols=ws,
                                         hold_windows=1, max_stations=4)
    y = _channel_output(x16, offsets, "fm", decim)
    _check_verdicts(y, offsets, "fm", wins, sess, ws * 2160, 1, 4)
    k = offs.index(m)
    diag = [(w["index"], offs[j], int(w["flags"][j]), w["rows"][j]["timing"], w["rows"][k]["timing"]) for w in wins
            for j in range(len(offs)) if w["rows"][j]["detected"]]
    assert [s["offset"] for s in sess] == [m], diag
    assert any(w["flags"][j] == bp.DETECTED | bp.LEAKAGE for w in wins for j in (k - 1, k + 1)), diag
    assert all(w["flags"][j] in (0, bp.DETECTED | bp.LEAKAGE) for w in wins for j in (k - 1, k + 1)), diag
    assert all(w["flags"][j] == 0 for w in wins for j in range(len(offs)) if abs(j - k) > 1), diag


# ---- AM: two stations (MA1, MA3)

AM2 = [(-20, 1, 1.0, 900, 0.0), (14, 2, 0.5, 1500, 20.0)]


@pytest.fixture(scope="module")
def am_band():
    from nrsc5_b200 import synth_am
    caps = [synth_am.make_am_ma1(nframes=3, seed=80 + i, lead_in=lead, psmi=psmi, cfo_hz=cfo, noise_lsb=0.0).cs16
            for i, (m, psmi, gain, lead, cfo) in enumerate(AM2)]
    n = min(c.size for c in caps) // 2
    N = 32 * n
    t = np.arange(N, dtype=np.float64)
    wide = np.zeros(N, dtype=np.complex128)
    for c, (m, psmi, gain, lead, cfo) in zip(caps, AM2):
        X = np.fft.fft(c[0:2 * n:2] + 1j * c[1:2 * n:2].astype(np.float64))
        Y = np.zeros(N, dtype=np.complex128)
        Y[: n // 2] = X[: n // 2]
        Y[-(n - n // 2):] = X[n // 2:]
        wide += np.fft.ifft(Y) * (32 * gain) * np.exp(2j * np.pi * ((80 * m) % 11907) / 11907.0 * t)
    rng = np.random.default_rng(9)
    wide += 60.0 * (rng.standard_normal(N) + 1j * rng.standard_normal(N))
    iq = np.empty(2 * N)
    iq[0::2], iq[1::2] = wide.real, wide.imag
    # seven windows of 96 symbols and a little: in the eighth, the channel 10 kHz beside the MA1 station once passes the
    # scan's phase rule, with a higher score than the station itself (include/nrsc5_b200.h, the band receiver's policy)
    return np.clip(np.rint(iq[: 2 * 32 * (7 * 96 * 270 + 1000)]), -32768, 32767).astype(np.int16)


@pytest.mark.gpu
def test_am_band(am_band):
    from nrsc5_b200 import engine as eng
    x = am_band
    offs = list(range(-30, 31))
    kw = dict(band="am", input_cs16=True, offsets=offs, window_symbols=96, hold_windows=2, max_stations=4)
    offsets, wins, sess, recs = _receive(x, **kw)
    y = _channel_output(x, offsets, "am", 32)
    _check_verdicts(y, offsets, "am", wins, sess, 96 * 270, 2, 4)
    assert sorted(s["offset"] for s in sess) == [-20, 14], [(s["offset"], s["n0"], s["n1"]) for s in sess]
    _check_records(y, sess, recs, "am")
    for raw in recs:
        assert any(t == eng.REC_SYNC for t, _ in eng.parse_records(raw))


@pytest.mark.gpu
def test_one_engine_stream_for_two_stations(am_band):
    x = am_band
    offs = list(range(-30, 31))
    offsets, wins, sess, recs = _receive(x, band="am", input_cs16=True, offsets=offs, window_symbols=96, hold_windows=2,
                                         max_stations=1)
    assert [s["offset"] for s in sess] == [-20]
    k = offs.index(14)
    assert all(w["flags"][k] & bp.NO_SLOT for w in wins if w["flags"][k] & bp.DETECTED and not w["flags"][k] & bp.LEAKAGE)
    assert any(w["flags"][k] & bp.NO_SLOT for w in wins)


# ---- a capture at 10 MS/s through the rate stage, D = 16

@pytest.mark.gpu
def test_rate_stage_session_and_records():
    from scipy.signal import resample, resample_poly
    from nrsc5_b200 import synth
    fs = 10000000
    cap = synth.make_fm(psmi=1, nframes=1, seed=44, lead_in=600, tail_blocks=2)
    z = cap.cu8.astype(np.float64) - 127.0
    y = resample_poly(z[0::2] + 1j * z[1::2], 1, 2)               # the station at 744 187.5 S/s
    n = int(y.size * fs / 744187.5)
    t = np.arange(n)
    rng = np.random.default_rng(3)
    w = resample(y, n) * 64.0 * np.exp(2j * np.pi * 400e3 * t / fs) + 30.0 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    x = np.empty(2 * n)
    x[0::2], x[1::2] = w.real, w.imag
    x = np.clip(np.rint(x), -32768, 32767).astype(np.int16)
    offs = [-6, -2, 4, 9]
    kw = dict(band="fm", decim=16, rate=fs, input_cs16=True, offsets=offs, window_symbols=64, hold_windows=2, max_stations=2)
    offsets, wins, sess, recs = _receive(x, pieces=[(0, 2 * 12345), (2 * 12345, x.size)], **kw)
    ych = _channel_output(x, offsets, "fm", 16, rate=fs)
    _check_verdicts(ych, offsets, "fm", wins, sess, 64 * 2160, 2, 2)
    assert [s["offset"] for s in sess] == [4]
    _check_records(ych, sess, recs, "fm")
