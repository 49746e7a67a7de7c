"""The wideband channeliser's AM band plan (include/nrsc5_b200.h: nrsc5b_chan_create_am*): one capture at
1 488 375 S/s -> 10 kHz channels at 46 511.72 S/s through a 512-tap bank.  CPU tier: the published tables (the
filter's measured response, the FM tables untouched), the numpy restatement (tests/chan_oracle_am.py) against its own
rules, the argument checks that need no device.  GPU tier: the kernel against the restatement bit for bit (cu8 and
cs16, the whole medium-wave grid), streamed against one-shot, a band of MA1 / MA3 stations 40 dB apart all decoding
through an AM engine, the feed into a running AM engine against the one-shot channeliser + nrsc5b_push_cs16 path, and
an FM handle next to an AM one.  The channeliser runs on TMA and wgmma, which the CPU emulation of the kernels does not
model: there is no emulated twin.

Run on the H100: all green."""
import ctypes
import hashlib

import numpy as np
import pytest

import chan_oracle
import chan_oracle_am as am
from nrsc5_b200 import channelizer as ch
from nrsc5_b200.engine import EngineError

RATE = ch.AM_WIDE_RATE
TAPS = ch.TAPS_AM
PERIOD, DECIM = ch.PERIOD, ch.DECIM
EINVAL = -2
BAND = list(range(-58, 60))                                      # 530 .. 1700 kHz around a 1110 kHz centre: 118 channels


def _full_range(rng, nvalues):
    x = rng.integers(-32768, 32768, nvalues, dtype=np.int16)
    x[rng.integers(0, nvalues, 64)] = -32768
    x[rng.integers(0, nvalues, 64)] = 32767
    return x


def _saturating_window(taps, k):
    """512 samples of +-32767 in the sign pattern of channel k's taps: Re(acc) = 32767 sum(|Wr| + |Wi|), v beyond int16."""
    x = np.empty(2 * TAPS, dtype=np.int16)
    x[0::2] = np.where(taps[k, :, 0] >= 0, 32767, -32767)
    x[1::2] = np.where(taps[k, :, 1] >= 0, -32767, 32767)
    return x


def _splits(n, rng, big=(20000, 200000)):
    """Cut points (input units: cu8 bytes or int16 values) into pushes of every awkward kind: empty, one sample, shorter
    than the filter, not a multiple of 64, large."""
    cuts, pos, i = [0], 0, 0
    while pos < n:
        step = [0, 2, 2 * int(rng.integers(1, TAPS)), 64 * int(rng.integers(1, 40)) + 2 * int(rng.integers(1, 32)),
                2 * int(rng.integers(*big))][i % 5]
        pos = min(n, pos + step)
        cuts.append(pos)
        i += 1
    return list(zip(cuts[:-1], cuts[1:]))


def _response_db(taps_k, nfft=1 << 18):
    """|H(f)| of one channel's integer taps W_k[u] in dB re its peak, on an nfft-point grid of the capture rate.  The
    taps are the time-reversed impulse response; the magnitude does not care."""
    w = taps_k[::-1, 0].astype(np.float64) + 1j * taps_k[::-1, 1].astype(np.float64)
    h = np.abs(np.fft.fft(w, nfft))
    return 20 * np.log10(np.maximum(h, 1e-9) / h.max()), np.fft.fftfreq(nfft, 1 / RATE)


# ---------------------------------------------------------------- CPU tier

def test_am_tables_filter_meets_its_figures_and_fm_tables_are_untouched():
    offs = [0, 1, -58, 59, 74, -74, 5]
    taps, ph = ch.make_tables(offs, band="am")
    assert taps.shape == (len(offs), TAPS, 2)
    fm_taps, fm_ph = ch.make_tables(list(range(-118, 119)))
    assert np.array_equal(ph, fm_ph)                             # one phasor table for both plans
    # the FM plan's tables as they were before the AM plan existed
    assert hashlib.sha256(fm_taps.tobytes() + fm_ph.tobytes()).hexdigest() == \
        "98b3e49ec32b4bc20a47213d8258869b353d4c324ce01750dc57229bb86eadf4"
    db, f = _response_db(taps[0])
    assert np.all(taps[0, :, 1] == 0)
    assert np.abs(db[np.abs(f) <= 15000]).max() <= 0.25
    assert db[np.abs(f) >= 31500].max() <= -80.0
    binw = RATE / db.size
    for k, m in enumerate(offs):
        dbk, _ = _response_db(taps[k])
        d = (f - 10000.0 * m + RATE / 2) % RATE - RATE / 2      # distance from the channel's centre, cyclic
        assert np.abs(dbk[np.abs(d) <= 15000]).max() <= 0.25, m
        assert dbk[np.abs(d) >= 31500].max() <= -80.0, m
        # channel 0's response moved by 10 m kHz: the -6 dB edges lie 23 kHz either side of it, centred within one bin
        inside = d[dbk >= -6.0]
        assert abs(inside.max() + inside.min()) / 2 <= binw and abs(inside.max() - inside.min() - 46000.0) <= 100.0, m
    # the bounds the kernel's 32-bit arithmetic needs
    s = np.abs(taps.astype(np.int64)).sum(axis=(1, 2))
    assert 128 * s.max() < 1 << 28 and np.abs(taps).max() <= 127 * 256 + 127


def test_am_restatement_outputs_carry_and_formats():
    rng = np.random.default_rng(2)
    offs = [0, -58, 59, 33]
    taps, ph = ch.make_tables(offs, band="am")
    for t in list(range(0, 1400)) + [10 ** 6 + k for k in range(70)]:
        n = am.outputs_of(t, TAPS)
        assert n == sum(1 for m in range(t // 32 + 1) if 32 * m + TAPS <= t)
        assert 0 <= t - 32 * n <= TAPS - 1 and (t < TAPS or t - 32 * n >= TAPS - 32)
        assert n == ch.stream_outputs(0, 2 * t, band="am") == ch.outputs(2 * t, band="am")
    assert ch.outputs(64 * 100, band="am") == 100 - 15 and ch.outputs(64 * 100) == 100 - 7
    assert ch.stream_outputs(511, 2, band="am") == 1 and ch.stream_outputs(512, 62, band="am") == 0
    cu8 = rng.integers(0, 256, 64 * 300 + 22, dtype=np.uint8)
    cu8[:64], cu8[64:128] = 0, 255
    x16 = (64 * (cu8.astype(np.int16) - 127)).astype(np.int16)
    want = am.channelize(cu8, offs, taps, ph)
    assert want.shape == (4, 2 * (300 - 15)) and np.abs(want).max() > 1000
    assert np.array_equal(am.channelize(x16, offs, taps, ph), want)
    # streamed == one-shot, for both formats
    for x in (cu8, _full_range(rng, 64 * 300 + 22)):
        parts = _splits(x.size, rng, big=(2000, 9000))
        outs = am.channelize_stream([x[a:b] for a, b in parts], offs, taps, ph)
        assert [o.shape[1] for o in outs] == [2 * ch.stream_outputs(a // 2, b - a, band="am") for a, b in parts]
        assert np.array_equal(np.concatenate(outs, axis=1), am.channelize(x, offs, taps, ph))
    # with the FM plan's tables and mixer step the restatement is the FM one
    fm_taps, fm_ph = ch.make_tables([7, -30])
    assert np.array_equal(am.channelize(cu8[: 64 * 300], [7, -30], fm_taps, fm_ph, mix_step=1600),
                          chan_oracle.channelize(cu8, [7, -30], fm_taps, fm_ph))


def test_am_v_saturates_on_full_scale_input():
    offs = [0, 37, -58]
    taps, ph = ch.make_tables(offs, band="am")
    for k in range(len(offs)):
        x = np.concatenate([_saturating_window(taps, k), np.zeros(64, dtype=np.int16)])
        acc = 32767 * int(np.abs(taps[k].astype(np.int64)).sum())
        assert (acc + (1 << 18)) >> 19 > 40000
        y = am.channelize(x, offs, taps, ph)
        assert y[k, 0] == (32767 * 32767 + (1 << 14)) >> 15 == 32766   # sat16(v) x conj(P[0]) = 32767


def test_am_argument_checks_without_a_device():
    L = ch._lib()
    taps = np.zeros((3, TAPS, 2), dtype=np.int16)
    ok = np.array([0, 74, -74], dtype=np.int32)
    assert L.nrsc5b_chan_make_tables_am(ok.ctypes.data, 3, taps.ctypes.data, None) == 0
    assert L.nrsc5b_chan_make_tables_am(ok.ctypes.data, 3, None, None) == 0
    for bad in ([0, 75, 1], [-75, 0, 1]):
        b = np.array(bad, dtype=np.int32)
        assert L.nrsc5b_chan_make_tables_am(b.ctypes.data, 3, taps.ctypes.data, None) == EINVAL
        h = ctypes.c_void_p()
        assert L.nrsc5b_chan_create_am(ctypes.byref(h), 0, b.ctypes.data, 3) == EINVAL and not h.value
        assert L.nrsc5b_chan_create_am_cs16(ctypes.byref(h), 0, b.ctypes.data, 3) == EINVAL and not h.value
    assert L.nrsc5b_chan_make_tables_am(None, 3, taps.ctypes.data, None) == EINVAL
    assert L.nrsc5b_chan_make_tables_am(ok.ctypes.data, 0, taps.ctypes.data, None) == EINVAL
    assert L.nrsc5b_chan_make_tables_am(ok.ctypes.data, -1, taps.ctypes.data, None) == EINVAL
    h = ctypes.c_void_p()
    assert L.nrsc5b_chan_create_am(None, 0, ok.ctypes.data, 3) == EINVAL
    assert L.nrsc5b_chan_create_am(ctypes.byref(h), 0, None, 3) == EINVAL
    assert L.nrsc5b_chan_create_am_cs16(ctypes.byref(h), 0, ok.ctypes.data, 0) == EINVAL
    assert L.nrsc5b_chan_outputs_am(1022) == 0 and L.nrsc5b_chan_outputs_am(1024) == 1 and L.nrsc5b_chan_outputs_am(64 * 50) == 35
    with pytest.raises(ValueError):
        ch.make_tables([0], band="lw")
    # the FM plan takes offsets the AM capture could not hold
    assert ch.make_tables([118, -118])[0].shape == (2, 256, 2)


def test_am_channelizer_needs_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    for cs16 in (False, True):
        with pytest.raises(EngineError):
            ch.Channelizer([0, 9], input_cs16=cs16, band="am")


# ---------------------------------------------------------------- GPU tier

def _random_offsets(rng, nch):
    return [-74] + [int(m) for m in rng.choice(np.arange(-73, 74), nch - 2, replace=False)] + [74]


# the whole band; a capture of exactly one filter length (one output); one output short of two tiles; a partial last
# group; past output 11907, where the mixer wraps
CASES = [("band", 32 * 700 + TAPS - 32), ("band", TAPS), (40, 32 * 126 + TAPS - 32), (33, 32 * 1031 + TAPS + 5),
         (5, 32 * 12100 + TAPS + 17)]


@pytest.mark.gpu
@pytest.mark.parametrize("cs16", [False, True], ids=["cu8", "cs16"])
@pytest.mark.parametrize("nch,nsamples", CASES)
def test_am_kernel_equals_the_restatement_bit_for_bit(nch, nsamples, cs16):
    rng = np.random.default_rng(60 + nsamples % 97)
    offs = BAND if nch == "band" else _random_offsets(rng, nch)
    with ch.Channelizer(offs, input_cs16=cs16, band="am") as c:
        taps, ph = c.tables()
        t2, p2 = ch.make_tables(offs, band="am")
        assert np.array_equal(taps, t2) and np.array_equal(ph, p2)
        if cs16:
            x = _full_range(rng, 2 * nsamples)
            for j, k in enumerate(range(0, len(offs), max(1, len(offs) // 4))):   # saturating windows for outputs 0, 16, ...
                if 2 * TAPS * (j + 1) <= x.size:
                    x[2 * TAPS * j: 2 * TAPS * (j + 1)] = _saturating_window(taps, k)
        else:
            x = rng.integers(0, 256, 2 * nsamples, dtype=np.uint8)
            x[:128], x[128:256] = 0, 255
        got = c.run(x)
    nout = am.outputs_of(nsamples, TAPS)
    assert got.shape == (len(offs), 2 * nout) and nout == ch.outputs(2 * nsamples, band="am")
    want = am.channelize(x, offs, taps, ph)
    if cs16:
        assert (np.abs(want.astype(np.int32)) >= 32766).any()    # both sat16s were at work
    bad = np.argwhere(got != want)
    assert bad.size == 0, f"{bad.shape[0]} of {got.size} values differ; first at (channel, value) {bad[:5].tolist()}"


@pytest.mark.gpu
def test_am_cs16_kernel_is_the_cu8_kernel_on_scaled_input():
    rng = np.random.default_rng(12)
    cu8 = rng.integers(0, 256, 64 * 2500, dtype=np.uint8)
    cu8[:64], cu8[64:128] = 0, 255
    x16 = (64 * (cu8.astype(np.int16) - 127)).astype(np.int16)
    with ch.Channelizer(BAND, band="am") as c8, ch.Channelizer(BAND, input_cs16=True, band="am") as c16:
        a, b = c8.run(cu8), c16.run(x16)
    assert a.shape == (118, 2 * (2500 - 15)) and np.array_equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("cs16", [False, True], ids=["cu8", "cs16"])
def test_am_streamed_kernel_equals_one_shot_bit_for_bit(cs16):
    """Random splits from host, page-locked and device memory; a push larger than the staging; reset."""
    import torch
    rng = np.random.default_rng(100 + cs16)
    offs = _random_offsets(rng, 35)
    n = 64 * 25001 + 38
    x = _full_range(rng, n) if cs16 else rng.integers(0, 256, n, dtype=np.uint8)
    parts = _splits(n, rng)
    sizes = [b - a for a, b in parts]
    assert 0 in sizes and 2 in sizes and any(0 < s < 2 * TAPS for s in sizes) and any(s % 64 for s in sizes)
    unit = x.itemsize
    with ch.Channelizer(offs, input_cs16=cs16, band="am") as c:
        taps, ph = c.tables()
        whole = c.run(x)
        got = [c.push(x[a:b]) for a, b in parts]
        assert c.pushed == n // 2
        c.reset()
        assert c.pushed == 0
        d_x, h_x = torch.from_numpy(x).cuda(), torch.from_numpy(x).pin_memory()
        nout = ch.outputs(n, band="am")
        d_out = torch.zeros((len(offs), 2 * nout + 64), dtype=torch.int16, device="cuda")
        col = 0
        for i, (a, b) in enumerate(parts):
            src = d_x if i % 2 else h_x
            col += 2 * c.push_device(src.data_ptr() + unit * a, b - a, d_out.data_ptr() + 2 * col, d_out.shape[1])
        torch.cuda.synchronize()
        assert col == 2 * nout
        # larger than the staging buffer (4 MiB of cu8; 2^22 samples of cs16), after a reset that drops a carry
        big = (9 << 20) + 6
        xb = np.tile(x, big // n + 1)[:big]
        c.reset()
        streamed = np.concatenate([c.push(xb[:302]), c.push(xb[302: big - 1000]), c.push(xb[big - 1000:])], axis=1)
        whole_b = c.run(xb)
    assert [g.shape[1] for g in got] == [2 * ch.stream_outputs(a // 2, b - a, band="am") for a, b in parts]
    assert np.array_equal(np.concatenate(got, axis=1), whole)
    assert np.array_equal(d_out[:, : 2 * nout].cpu().numpy(), whole)
    assert np.array_equal(whole[:, : 2 * 3000], am.channelize(x[: 2 * (32 * 2999 + TAPS)], offs, taps, ph))
    assert np.array_equal(streamed, whole_b)
    nb = ch.outputs(big, band="am")
    tail = am.channelize(xb[64 * (nb - 300):], offs, taps, ph, n0=nb - 300)
    assert np.array_equal(streamed[:, 2 * (nb - 300):], tail)


# ---- a band of stations through the channeliser into an AM engine

# (offset in 10 kHz steps, level in dB re the generator's default, MA3?)  -53 and -58 are five channels apart: the
# station at -53 aliases onto -58 after the decimation by 32 (50 kHz - 46.5 kHz = 3.5 kHz off its centre) and is 30 dB
# stronger.  Channels -20 and 40 hold no station.
STATIONS = [(-58, -37.0, False), (-53, -7.0, False), (0, 3.0, True), (17, -20.0, False), (31, -30.0, True), (59, -37.0, False)]
OFFS = [m for m, _, _ in STATIONS] + [-20, 40]
NFRAMES = 7


def _band_capture(cs16=True):
    from nrsc5_b200 import synth_am
    caps = [synth_am.make_am_ma1(nframes=NFRAMES, seed=300 + i, lead_in=200 + 150 * i, cfo_hz=0.3 * (i - 2), psmi=2 if ma3 else 1)
            for i, (_, _, ma3) in enumerate(STATIONS)]
    if cs16:
        st = [(c.cs16, m, 10 ** (db / 20)) for c, (m, db, _) in zip(caps, STATIONS)]
        return synth_am.make_am_band(st, cs16=True, noise_lsb=3.0), caps
    # 8 bits cannot hold 40 dB between stations: three of them, at equal level, carrier 24 LSB
    st = [(c.cs16, m, 24.0 / 10000.0) for c, (m, _, _) in zip(caps, STATIONS)][1:4]
    return synth_am.make_am_band(st, cs16=False, noise_lsb=1.0), caps[1:4]


def _am_engine(nstreams, capacity):
    import nrsc5_b200
    e = nrsc5_b200.Engine(nstreams=nstreams, input_capacity=capacity, log_capacity=8 << 20, mode="am", input_cs16=True)
    e.enable_l2()
    return e


def _drain(e, s):
    """The stream's new records, every REC_L2 moved behind its frame and expanded into its events: within one
    nrsc5b_process the engine logs the L2 records after the L1 ones, so their place depends on how the input was cut
    into calls, the order of the reference's calls does not."""
    from nrsc5_b200 import engine as eng
    return eng.with_l2_in_call_order(e.drain_raw(s))


def _one_shot(x, offs, cs16):
    """nrsc5b_chan_run on the whole capture, nrsc5b_push_cs16 of every channel, one nrsc5b_process."""
    with ch.Channelizer(offs, input_cs16=cs16, band="am") as c:
        y = c.run(x)
    with _am_engine(len(offs), 2 * y.shape[1] + 4096) as e:
        for s in range(len(offs)):
            e.push_cs16(s, y[s])
        e.process()
        recs = [_drain(e, s) for s in range(len(offs))]
    return y, recs


@pytest.fixture(scope="module")
def band():
    x, caps = _band_capture()
    y, recs = _one_shot(x, OFFS, True)
    return x, caps, y, recs


def _pack(b):
    return np.packbits(np.asarray(b, dtype=np.uint8)).tobytes()


def _check_station(recs, y_row, cap, ma3):
    """The stream's P1 / P3 / PIDS PDUs are frames the generator put in, and its records are what the AM oracle decodes
    from the channeliser's output for that channel."""
    import port
    from nrsc5_b200 import engine as eng
    import test_gpu_am
    frames = [r for t, r in recs if t == eng.REC_FRAME]
    p1 = [r["bits"] for r in frames if r["lc"] == 0 and r["nbits"] == 3750]
    p3 = [r["bits"] for r in frames if r["lc"] == 1 and r["nbits"] == (30000 if ma3 else 24000)]
    pids = [r["bits"] for t, r in recs if t == eng.REC_PIDS]
    gen_p1 = {_pack(b) for fr in cap.p1_frames.values() for b in fr}
    gen_p3 = {_pack(b) for b in cap.p3_frames.values()}
    gen_pids = {_pack(b) for b in cap.pids_frames}
    assert len(p1) >= 8 and all(b in gen_p1 for b in p1)
    assert len(p3) >= 1 and all(b in gen_p3 for b in p3)
    assert len(pids) >= 16 and all(b in gen_pids for b in pids)
    assert test_gpu_am.digest(recs) == test_gpu_am.oracle_digest(port.decode_am(y_row))


@pytest.mark.gpu
def test_am_band_of_stations_40_db_apart_all_decode(band):
    from nrsc5_b200 import engine as eng
    x, caps, y, recs = band
    assert 16000 < np.abs(x.astype(np.int32)).max() < 32767      # the strong station fills the 16 bits, nothing clips
    taps, ph = ch.make_tables(OFFS, band="am")
    assert np.array_equal(y[:, : 2 * 3000], am.channelize(x[: 2 * (32 * 2999 + TAPS)], OFFS, taps, ph))
    for s, (m, db, ma3) in enumerate(STATIONS):
        _check_station(recs[s], y[s], caps[s], ma3)
    for s in range(len(STATIONS), len(OFFS)):                    # the empty channels: noise in, no frames out
        assert np.abs(y[s]).max() > 0
        assert not [1 for t, r in recs[s] if t in (eng.REC_FRAME, eng.REC_PIDS)]


@pytest.mark.gpu
def test_am_cu8_band_decodes():
    x, caps = _band_capture(cs16=False)
    offs = OFFS[1:4]
    y, recs = _one_shot(x, offs, False)
    for s in range(3):
        _check_station(recs[s], y[s], caps[s], STATIONS[1 + s][2])


def _without_positions(recs):
    """REC_BLOCK carries the block's start in the stream's input buffer, which a trim moves; everything else must agree."""
    from nrsc5_b200 import engine as eng
    return [(t, {k: v for k, v in r.items() if not (t == eng.REC_BLOCK and k == "start")}) for t, r in recs]


def _ragged(n, seed):
    rng = np.random.default_rng(seed)
    cuts, pos = [0], 0
    while pos < n:
        pos = min(n, pos + (2 * int(rng.integers(1, 300)) if rng.random() < 0.2 else 2 * int(rng.integers(1 << 19, 3 << 20))))
        cuts.append(pos)
    return list(zip(cuts[:-1], cuts[1:]))


@pytest.mark.gpu
def test_am_feed_with_permuted_streams(band):
    x, caps, y, ref = band
    perm = [3, 0, 7, 1, 6, 2, 5, 4]
    got = [[] for _ in OFFS]
    with ch.Channelizer(OFFS, input_cs16=True, band="am") as c, _am_engine(len(OFFS), 2 * y.shape[1] + 4096) as e:
        for a, b in _ragged(x.size, 1):
            c.feed(e, x[a:b], streams=perm)                      # channel k -> stream perm[k]
            e.process()
            for k in range(len(OFFS)):
                got[k] += _drain(e, perm[k])
    assert got == ref


@pytest.mark.gpu
def test_am_feed_into_small_input_buffers_trims(band):
    x, caps, y, ref = band
    cap = 1 << 20                                                # each channel's cs16 takes about 1.9 MB
    assert 2 * y.shape[1] > cap
    recs = [[] for _ in OFFS]
    with ch.Channelizer(OFFS, input_cs16=True, band="am") as c, _am_engine(len(OFFS), cap) as e:
        for a, b in _ragged(x.size, 2):
            c.feed(e, x[a:b])
            e.process()
            for s in range(len(OFFS)):
                recs[s] += _drain(e, s)
    assert [_without_positions(r) for r in recs] == [_without_positions(r) for r in ref]


@pytest.mark.gpu
def test_am_feed_back_pressure_is_all_or_nothing(band):
    """Pushes without processing until the engine is full: the push that gets NRSC5B_EFULL takes nothing, neither in
    the channeliser nor in the engine, and the same values go in after nrsc5b_process."""
    import torch
    x, caps, y, ref = band
    host = torch.from_numpy(x).pin_memory()
    step = 2 << 20                                               # int16 values per push: 32768 outputs, 128 KB per stream
    recs, refused = [[] for _ in OFFS], 0
    with ch.Channelizer(OFFS, input_cs16=True, band="am") as c, _am_engine(len(OFFS), 1 << 19) as e:
        pos, processing = 0, False
        while pos < x.size:
            n = min(step, x.size - pos)
            before = c.pushed
            try:
                c.feed(e, (host.data_ptr() + 2 * pos, n))
            except EngineError as ex:
                assert "EFULL" in str(ex) and not processing
                assert c.pushed == before
                refused += 1
                processing = True
                e.process()
                for s in range(len(OFFS)):
                    recs[s] += _drain(e, s)
                c.feed(e, (host.data_ptr() + 2 * pos, n))
            pos += n
            if processing:
                e.process()
                for s in range(len(OFFS)):
                    recs[s] += _drain(e, s)
        e.process()
        for s in range(len(OFFS)):
            recs[s] += _drain(e, s)
        torch.cuda.synchronize()
    assert refused == 1
    assert [_without_positions(r) for r in recs] == [_without_positions(r) for r in ref]


@pytest.mark.gpu
def test_am_feed_takes_exactly_the_matching_engine():
    """An FM handle on an AM engine, an AM handle on an FM engine, an AM engine made for cu8 input, an attached input,
    bad stream tables: NRSC5B_EINVAL, and a following valid feed goes on as if they had not been made."""
    import torch
    import nrsc5_b200
    rng = np.random.default_rng(3)
    offs = [5, -60]
    x = _full_range(rng, 64 * 2000 + 14)
    with ch.Channelizer(offs, input_cs16=True, band="am") as w:
        want = np.concatenate([w.push(x[:1000]), w.push(x[1000:])], axis=1)
    with ch.Channelizer(offs, input_cs16=True) as w:
        want_fm = np.concatenate([w.push(x[:1000]), w.push(x[1000:])], axis=1)
    attached = torch.zeros((2, 1 << 14), dtype=torch.int16, device="cuda")
    with ch.Channelizer(offs, input_cs16=True, band="am") as c, ch.Channelizer(offs, input_cs16=True) as fm_c, \
            nrsc5_b200.Engine(nstreams=3, input_capacity=1 << 20, log_capacity=1 << 16, mode="am", input_cs16=True) as e, \
            nrsc5_b200.Engine(nstreams=2, input_capacity=1 << 16, input_cs16=True) as fm, \
            nrsc5_b200.Engine(nstreams=2, input_capacity=1 << 16, mode="am", input_cs16=False) as am_cu8, \
            nrsc5_b200.Engine(nstreams=2, input_capacity=1 << 16, mode="am", input_cs16=True) as am_att:
        am_att.attach_device_input(attached.data_ptr(), 2 << 14, 0)
        first, first_fm = c.push(x[:1000]), fm_c.push(x[:1000])
        bad = [(c, fm, None), (c, am_cu8, None), (c, am_att, None), (c, e, [1, 1]), (c, e, [0, 3]), (c, e, [-1, 0]), (fm_c, e, None)]
        for c_, e_, streams in bad:
            with pytest.raises(EngineError, match="EINVAL"):
                c_.feed(e_, x[1000:], streams=streams)
            assert c_.pushed == 500
        with pytest.raises(EngineError, match="EINVAL"):
            c.feed(e, x[1000:1001])
        with ch.Channelizer([0, 1, 2, 3], input_cs16=True, band="am") as wide:   # more channels than the engine has streams
            with pytest.raises(EngineError, match="EINVAL"):
                wide.feed(e, x)
        torch.cuda.synchronize()
        c.feed(e, x[1000:60000], streams=[2, 0])
        fm_c.feed(fm, x[1000:60000])
        e.process()
        assert c.pushed == 30000
        rest, rest_fm = c.push(x[60000:]), fm_c.push(x[60000:])
    assert np.array_equal(first, want[:, : first.shape[1]])
    assert np.array_equal(rest, want[:, 2 * ch.stream_outputs(0, 60000, band="am"):])
    assert np.array_equal(first_fm, want_fm[:, : first_fm.shape[1]])
    assert np.array_equal(rest_fm, want_fm[:, 2 * ch.stream_outputs(0, 60000):])


@pytest.mark.gpu
def test_fm_and_am_handles_side_by_side():
    """Both plans and both formats alive in one process, used in turn: each gives its own definition's outputs."""
    import chan_oracle_cs16
    rng = np.random.default_rng(21)
    cu8 = rng.integers(0, 256, 64 * 1200, dtype=np.uint8)
    x16 = _full_range(rng, 64 * 1200)
    fm_offs, am_offs = [-118, 3, 118], [-58, 3, 59]
    with ch.Channelizer(fm_offs) as f8, ch.Channelizer(am_offs, band="am") as a8, \
            ch.Channelizer(fm_offs, input_cs16=True) as f16, ch.Channelizer(am_offs, input_cs16=True, band="am") as a16:
        got = [f8.run(cu8), a8.run(cu8), f16.run(x16), a16.run(x16), a8.push(cu8), f8.push(cu8)]
        assert f8.tables()[0].shape[1] == 256 and a8.tables()[0].shape[1] == 512
    ft, fp = ch.make_tables(fm_offs)
    at, ap = ch.make_tables(am_offs, band="am")
    assert np.array_equal(got[0], chan_oracle.channelize(cu8, fm_offs, ft, fp))
    assert np.array_equal(got[1], am.channelize(cu8, am_offs, at, ap))
    assert np.array_equal(got[2], chan_oracle_cs16.channelize_cs16(x16, fm_offs, ft, fp))
    assert np.array_equal(got[3], am.channelize(x16, am_offs, at, ap))
    assert np.array_equal(got[4], got[1]) and np.array_equal(got[5], got[0])
