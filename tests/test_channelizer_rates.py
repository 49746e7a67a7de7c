"""The wideband channeliser's FM plans for 11.907 and 5.9535 MS/s captures (include/nrsc5_b200.h:
nrsc5b_chan_create_fm, decimation D = 16 and 8).  CPU tier: the tables per D (unit DC gain at 2^14 D, flatness, stop
band, int8 tap bytes, the 32-bit epilogue bound over the whole offset range), D = 32 being the FM plan bit for bit, the
argument checks, and the numpy restatement (tests/chan_oracle_rates.py) on known signals, on scaled cu8 and streamed.
GPU tier: the kernel against the restatement bit for bit, cs16 against cu8, streamed against one-shot, and synthetic
stations in one capture decoding through an FM cs16 engine, one-shot and fed."""
import ctypes

import numpy as np
import pytest

import chan_oracle
import chan_oracle_rates as rates
from nrsc5_b200 import channelizer as ch
from nrsc5_b200.engine import EngineError

EINVAL = -2
MAX_OFF = {16: 59, 8: 29}
DS = [16, 8]


def _full_range(rng, nvalues):
    x = rng.integers(-32768, 32768, nvalues, dtype=np.int16)
    x[rng.integers(0, nvalues, 64)] = -32768
    x[rng.integers(0, nvalues, 64)] = 32767
    return x


def _offsets(rng, nch, decim):
    """nch distinct offsets over the plan's whole range, both ends included when nch >= 2."""
    m = MAX_OFF[decim]
    if nch == 2 * m + 1:
        return list(range(-m, m + 1))
    if nch == 1:
        return [int(rng.integers(-m, m + 1))]
    inner = [int(v) for v in rng.choice(np.arange(-m + 1, m), nch - 2, replace=False)]
    return [-m] + inner + [m]


def _splits(nvalues, rng, big=(20000, 200000)):
    """Cut points of a capture into pushes of every awkward kind: empty, one sample, shorter than the filter, not a
    multiple of 32 samples, large."""
    cuts, pos, i = [0], 0, 0
    while pos < nvalues:
        step = [0, 2, 2 * int(rng.integers(1, 256)), 64 * int(rng.integers(1, 40)) + 2 * int(rng.integers(1, 32)),
                2 * int(rng.integers(*big))][i % 5]
        pos = min(nvalues, pos + step)
        cuts.append(pos)
        i += 1
    return list(zip(cuts[:-1], cuts[1:]))


def _tone(m, amp, n, decim, phase=0.3):
    t = np.arange(n)
    x = amp * np.exp(1j * (2 * np.pi * m * 100e3 / ch.wide_rate(decim) * t + phase))
    a = np.empty(2 * n, dtype=np.uint8)
    a[0::2] = np.clip(np.rint(x.real + 127), 0, 255)
    a[1::2] = np.clip(np.rint(x.imag + 127), 0, 255)
    return a


# ---------------------------------------------------------------- CPU tier

@pytest.mark.parametrize("decim", DS)
def test_tables_per_rate(decim):
    m = MAX_OFF[decim]
    offs = list(range(-m, m + 1))
    taps, ph = ch.make_tables(offs, decim=decim)
    assert taps.shape == (len(offs), 256, 2)
    _, ph32 = ch.make_tables([0])
    assert np.array_equal(ph, ph32)                                        # the one phasor table
    h = taps[m, :, 0].astype(np.float64)                                   # channel 0: no mixing, real taps
    assert np.all(taps[m, :, 1] == 0) and abs(h.sum() - 2 ** 14 * decim) < 64   # unit DC gain at the 2^14 D scale
    H = np.abs(np.fft.fft(h, 1 << 16)) / h.sum()
    f = np.fft.fftfreq(1 << 16, 1 / ch.wide_rate(decim))
    assert H[np.abs(f) <= 200e3].min() > 0.97                              # the FM plan's bounds ...
    assert H[np.abs(f) >= 544e3].max() < 10 ** (-55 / 20)
    assert np.abs(20 * np.log10(H[np.abs(f) <= 200e3])).max() < 0.01      # ... and the figures this plan reaches
    assert H[np.abs(f) >= 544e3].max() < 10 ** (-78 / 20)
    t = taps.astype(np.int64)
    assert np.abs(t).max() <= 127 * 256 + 127                             # both bytes of every tap are int8
    assert 15000 < np.abs(h).max() < 17000                                # the peak stays near 2^14 for every D
    s_cu8, _ = rates.shifts(decim)
    S = (np.abs(t[:, :, 0]) + np.abs(t[:, :, 1])).sum(axis=1)
    assert (128 * S).max() < 2 ** 28                                      # the cu8 epilogue and the cs16 combine
    assert (128 * S).max() < 2 ** (15 + s_cu8)                             # |v| < 2^15: the rotation stays in 32 bits
    mag = np.hypot(taps[0, :, 0].astype(float), taps[0, :, 1].astype(float))
    assert np.abs(mag - np.abs(h)).max() <= 1.5                            # a mixed channel: the prototype times a phasor


def test_decim_32_tables_are_the_fm_plan():
    offs = list(range(-118, 119))
    t32, p32 = ch.make_tables(offs)
    L = ch._lib()
    off = np.ascontiguousarray(offs, dtype=np.int32)
    taps = np.empty_like(t32)
    ph = np.empty_like(p32)
    assert L.nrsc5b_chan_make_tables_fm(32, off.ctypes.data, off.size, taps.ctypes.data, ph.ctypes.data) == 0
    assert np.array_equal(taps, t32) and np.array_equal(ph, p32)
    for nbytes in (0, 64, 512, 64 * 1000, 64 * 12345):
        assert L.nrsc5b_chan_outputs_fm(32, nbytes) == L.nrsc5b_chan_outputs(nbytes)


def test_argument_checks_without_a_device():
    L = ch._lib()
    vp = ctypes.c_void_p
    off = np.array([0, 5], dtype=np.int32)
    taps = np.zeros((2, 256, 2), dtype=np.int16)
    for d in (0, 1, 4, 24, 64, -16):
        assert L.nrsc5b_chan_make_tables_fm(d, off.ctypes.data, 2, taps.ctypes.data, None) == EINVAL
        assert L.nrsc5b_chan_outputs_fm(d, 6400) == EINVAL
        h = vp()
        assert L.nrsc5b_chan_create_fm(ctypes.byref(h), 0, d, off.ctypes.data, 2) == EINVAL
        assert L.nrsc5b_chan_create_fm_cs16(ctypes.byref(h), 0, d, off.ctypes.data, 2) == EINVAL
        assert not h.value
    for d, m in MAX_OFF.items():
        for bad in ([m + 1], [-m - 1], [0, 3, m + 1]):
            b = np.array(bad, dtype=np.int32)
            assert L.nrsc5b_chan_make_tables_fm(d, b.ctypes.data, b.size, None, None) == EINVAL
            h = vp()
            assert L.nrsc5b_chan_create_fm(ctypes.byref(h), 0, d, b.ctypes.data, b.size) == EINVAL
            assert L.nrsc5b_chan_create_fm_cs16(ctypes.byref(h), 0, d, b.ctypes.data, b.size) == EINVAL
        ok = np.array([-m, m], dtype=np.int32)
        assert L.nrsc5b_chan_make_tables_fm(d, ok.ctypes.data, 2, None, None) == 0
        assert L.nrsc5b_chan_make_tables_fm(d, ok.ctypes.data, 0, None, None) == EINVAL
        assert L.nrsc5b_chan_make_tables_fm(d, None, 2, None, None) == EINVAL
    for nbytes in (0, 64, 448, 512, 576, 64 * 1000):
        assert L.nrsc5b_chan_outputs_fm(16, nbytes) == max(nbytes // 32 - 15, 0)
        assert L.nrsc5b_chan_outputs_fm(8, nbytes) == max(nbytes // 16 - 31, 0)
    with pytest.raises(ValueError):
        ch.make_tables([0], band="am", decim=16)
    with pytest.raises(ValueError):
        ch.outputs(6400, decim=4)
    with pytest.raises(ValueError):
        ch.stream_outputs(0, 6400, band="am", decim=8)
    with pytest.raises(ValueError):
        ch.Channelizer([0], band="am", decim=16)
    with pytest.raises(ValueError):
        ch.wide_rate(24)
    assert ch.wide_rate() == ch.WIDE_RATE and ch.wide_rate(16) == 11907000.0 and ch.wide_rate(8) == 5953500.0


@pytest.mark.parametrize("decim", DS)
def test_restatement_moves_a_tone_to_dc_and_rejects_the_neighbour(decim):
    m = 17 if decim == 16 else 9
    offs = [m, m - 6]
    taps, ph = ch.make_tables(offs, decim=decim)
    y = rates.channelize(_tone(m, 50.0, decim * 1200, decim), offs, taps, ph, decim).astype(np.float64)
    z0 = y[0, 0::2] + 1j * y[0, 1::2]
    z1 = y[1, 0::2] + 1j * y[1, 1::2]
    assert abs(np.abs(z0).mean() - 50.0 * 64) < 0.02 * 50 * 64            # unit gain: 64 LSB per input LSB
    assert np.abs(z0 - z0.mean()).max() < 0.02 * 50 * 64                  # a constant: the tone sits at DC
    # rejected by the channel 600 kHz away (stop band): what is left is the rounding noise of the 8-bit input that falls
    # into that channel, a larger share of the capture's band than at D = 32, so its rms is bounded here, not its peak
    assert np.sqrt(np.mean(np.abs(z1) ** 2)) < 50.0 * 64 * 10 ** (-48 / 20)


@pytest.mark.parametrize("decim", [32] + DS)
def test_restatement_cs16_on_scaled_cu8_is_cu8(decim):
    rng = np.random.default_rng(decim)
    offs = _offsets(rng, 4, decim) if decim != 32 else [-118, 5, 60, 118]
    taps, ph = ch.make_tables(offs, decim=decim)
    cu8 = rng.integers(0, 256, 64 * 700, dtype=np.uint8)
    cu8[:64], cu8[64:128] = 0, 255
    x16 = (64 * (cu8.astype(np.int16) - 127)).astype(np.int16)
    want = rates.channelize(cu8, offs, taps, ph, decim, n0=11800)
    assert np.array_equal(rates.channelize(x16, offs, taps, ph, decim, n0=11800), want)
    if decim == 32:                                                        # and at D = 32 it is the FM plan's restatement
        assert np.array_equal(want, chan_oracle.channelize(cu8, offs, taps, ph, n0=11800))


@pytest.mark.parametrize("decim", DS)
def test_restated_stream_equals_one_shot(decim):
    rng = np.random.default_rng(7 + decim)
    offs = _offsets(rng, 3, decim)
    taps, ph = ch.make_tables(offs, decim=decim)
    nvalues = 2 * int(rng.integers(60000, 90000))
    x = _full_range(rng, nvalues)
    parts = _splits(nvalues, rng)
    outs = rates.channelize_stream([x[a:b] for a, b in parts], offs, taps, ph, decim)
    assert [o.shape[1] for o in outs] == [2 * ch.stream_outputs(a // 2, b - a, decim=decim) for a, b in parts]
    assert np.array_equal(np.concatenate(outs, axis=1), rates.channelize(x, offs, taps, ph, decim))


def test_channelizer_needs_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    for d in DS:
        for cs16 in (False, True):
            with pytest.raises(EngineError):
                ch.Channelizer([0, 9], input_cs16=cs16, decim=d)


# ---------------------------------------------------------------- GPU tier

def _input(rng, nsamples, cs16):
    return _full_range(rng, 2 * nsamples) if cs16 else rng.integers(0, 256, 2 * nsamples, dtype=np.uint8)


@pytest.mark.gpu
@pytest.mark.parametrize("cs16", [False, True])
@pytest.mark.parametrize("decim", DS)
@pytest.mark.parametrize("nch,nout", [(1, 1), (33, 64 * 5 + 17), ("full", 12100), ("full", 1)])
def test_kernel_equals_the_restatement_bit_for_bit(nch, nout, decim, cs16):
    """One output, a partial tile and more than one channel group, the whole offset range with the mixer wrapping past
    output 11907.  The capture is 32 samples longer than the outputs need (not whole 64-byte rows for cs16)."""
    rng = np.random.default_rng(nout + decim + (1000 if cs16 else 0))
    n = 2 * MAX_OFF[decim] + 1 if nch == "full" else nch
    offs = _offsets(rng, n, decim)
    nsamples = decim * (nout - 1) + 256 + (7 if cs16 else 0)
    x = _input(rng, nsamples, cs16)
    with ch.Channelizer(offs, input_cs16=cs16, decim=decim) as c:
        taps, ph = c.tables()
        t2, p2 = ch.make_tables(offs, decim=decim)
        assert np.array_equal(taps, t2) and np.array_equal(ph, p2)
        if not cs16:
            x = np.concatenate([x, rng.integers(0, 256, (-x.size) % 64, dtype=np.uint8)])
        got = c.run(x)
    want = rates.channelize(x, offs, taps, ph, decim)
    assert got.shape == want.shape and got.shape[1] >= 2 * nout
    bad = np.argwhere(got != want)
    assert bad.size == 0, f"{bad.shape[0]} of {got.size} values differ; first at (channel, value) {bad[:5].tolist()}: " \
                          f"got {got[tuple(bad[0])]} want {want[tuple(bad[0])]}"


@pytest.mark.gpu
@pytest.mark.parametrize("decim", DS)
def test_cs16_kernel_on_scaled_cu8_equals_the_cu8_kernel(decim):
    rng = np.random.default_rng(21 + decim)
    offs = _offsets(rng, 35, decim)
    cu8 = rng.integers(0, 256, 64 * 20000, dtype=np.uint8)
    x16 = (64 * (cu8.astype(np.int16) - 127)).astype(np.int16)
    parts = _splits(x16.size, rng)
    with ch.Channelizer(offs, decim=decim) as c8, ch.Channelizer(offs, input_cs16=True, decim=decim) as c16:
        want = c8.run(cu8)
        assert np.array_equal(c16.run(x16), want)
        s8 = np.concatenate([c8.push(cu8[a:b]) for a, b in parts], axis=1)
        s16 = np.concatenate([c16.push(x16[a:b]) for a, b in parts], axis=1)
    assert np.array_equal(s8, want) and np.array_equal(s16, want)


@pytest.mark.gpu
@pytest.mark.parametrize("cs16", [False, True])
def test_decim_32_through_the_new_creator_is_the_fm_plan(cs16):
    rng = np.random.default_rng(5)
    offs = np.ascontiguousarray([-118, -3, 0, 41, 118], dtype=np.int32)
    x = _input(rng, 32 * 3000, cs16)
    L = ch._lib()
    h = ctypes.c_void_p()
    create = L.nrsc5b_chan_create_fm_cs16 if cs16 else L.nrsc5b_chan_create_fm
    assert create(ctypes.byref(h), 0, 32, offs.ctypes.data, offs.size) == 0
    try:
        nout = ch.outputs(x.size)
        got = np.empty((offs.size, 2 * nout), dtype=np.int16)
        run = L.nrsc5b_chan_run_cs16 if cs16 else L.nrsc5b_chan_run
        assert run(h, x.ctypes.data, x.size, got.ctypes.data) == 0
    finally:
        L.nrsc5b_chan_destroy(h)
    with ch.Channelizer(offs, input_cs16=cs16) as c:
        assert np.array_equal(got, c.run(x))


@pytest.mark.gpu
@pytest.mark.parametrize("cs16", [False, True])
@pytest.mark.parametrize("decim", DS)
def test_streamed_equals_one_shot_from_every_kind_of_memory(decim, cs16):
    """Awkward splits from pageable, page-locked and device memory, the mixer wrapping inside the stream; then reset and
    the same again."""
    import torch
    rng = np.random.default_rng(200 + decim + cs16)
    offs = _offsets(rng, 33, decim)
    nvalues = 2 * (decim * 13001 + 19)
    x = _input(rng, nvalues // 2, cs16)
    item = 2 if cs16 else 1
    parts = _splits(nvalues, rng)
    nout = ch.stream_outputs(0, nvalues, decim=decim)
    d_x = torch.from_numpy(x).cuda()
    h_x = torch.from_numpy(x).pin_memory()
    with ch.Channelizer(offs, input_cs16=cs16, decim=decim) as c:
        taps, ph = c.tables()
        whole = rates.channelize(x, offs, taps, ph, decim)
        assert whole.shape[1] == 2 * nout
        for rep in range(2):
            if rep:
                c.reset()
                assert c.pushed == 0
            d_out = torch.zeros((len(offs), 2 * nout + 64), dtype=torch.int16, device="cuda")
            col = 0
            for i, (a, b) in enumerate(parts):
                if i % 3 == 0:
                    got = c.push(x[a:b])                              # pageable
                    d_out[:, col: col + got.shape[1]] = torch.from_numpy(got).cuda()
                    col += got.shape[1]
                else:
                    src = d_x if i % 3 == 1 else h_x
                    n = c.push_device(src.data_ptr() + item * a, b - a, d_out.data_ptr() + 2 * col, d_out.shape[1])
                    col += 2 * n
            torch.cuda.synchronize()
            assert col == 2 * nout and c.pushed == nvalues // 2
            streamed = d_out[:, : 2 * nout].cpu().numpy()
            bad = np.argwhere(streamed != whole)
            assert bad.size == 0, f"pass {rep}: {bad.shape[0]} values differ; first at {bad[:5].tolist()}"


@pytest.mark.gpu
@pytest.mark.parametrize("cs16", [False, True])
def test_capture_larger_than_the_scratch(cs16):
    """D = 8, 2^22 + 300 000 samples: the one-shot cs16 entry goes through its planes in pieces of 2^19 outputs, a push
    larger than the staging buffer goes through it in pieces; both equal the restatement at the start, across the
    piece boundary and at the end."""
    import torch
    decim = 8
    rng = np.random.default_rng(31)
    offs = [0, 29, -29, 11, -17]
    nvalues = 2 * ((1 << 22) + 300000)
    x = _input(rng, nvalues // 2, cs16)
    nout = ch.outputs(nvalues, decim=decim)
    stride = 2 * nout + 32
    d_x = torch.from_numpy(x).cuda()
    with ch.Channelizer(offs, input_cs16=cs16, decim=decim) as c:
        taps, ph = c.tables()
        d_out = torch.zeros((len(offs), stride), dtype=torch.int16, device="cuda")
        c.run_device(d_x.data_ptr(), nvalues, d_out.data_ptr(), stride)
        torch.cuda.synchronize()
        one = d_out[:, : 2 * nout].cpu().numpy()
        got = np.concatenate([c.push(x[:302]), c.push(x[302: nvalues - 1000]), c.push(x[nvalues - 1000:])], axis=1)
    assert np.array_equal(got, one)
    for n0, n in ((0, 600), ((1 << 19) - 300, 600), (nout - 300, 300)):
        want = rates.channelize(x[2 * decim * n0: 2 * (decim * (n0 + n - 1) + 256)], offs, taps, ph, decim, n0=n0)
        assert np.array_equal(one[:, 2 * n0: 2 * (n0 + n)], want), f"outputs {n0} .. {n0 + n - 1}"


# ---- synthetic stations in one capture, one-shot into an engine and fed straight into it

# (offset in 100 kHz, amplitude, generator seed, lead-in) per D: a strong MP1 station near full scale, a weak one 48 dB
# under it, and a neighbour 200 kHz from the weak one; the same stations at every D, so that only the plan differs
STATIONS = {d: [(11, 250.0, 90, 40), (-23, 1.0, 91, 540), (-21, 60.0, 93, 1540)] for d in (32, 16, 8)}


def _band_capture(decim):
    """The stations' 1 488 375 S/s captures interpolated by D / 2 (band-limited, on the GPU) into one cs16 capture at
    D x 744 187.5 S/s with a little noise."""
    import math
    import torch
    from nrsc5_b200 import synth
    st = STATIONS[decim]
    caps = [synth.make_fm_mp1(nframes=1, seed=seed, lead_in=lead, tail_blocks=3) for _, _, seed, lead in st]
    n = min(c.cu8.size for c in caps) // 2
    up = decim // 2
    N = n * up
    wide = torch.zeros(N, dtype=torch.complex64, device="cuda")
    t = torch.arange(N, dtype=torch.float64, device="cuda")
    for c, (m, s, _, _) in zip(caps, st):
        xi = torch.from_numpy(c.cu8[: 2 * n].astype(np.float32) - 127.0).cuda().view(-1, 2)
        X = torch.fft.fft(torch.complex(xi[:, 0].contiguous(), xi[:, 1].contiguous()))
        Y = torch.zeros(N, dtype=torch.complex64, device="cuda")
        Y[: n // 2] = X[: n // 2]
        Y[-(n - n // 2):] = X[n // 2:]
        y = torch.fft.ifft(Y) * (up * s)
        phase = torch.remainder(t * (m * 100e3 / ch.wide_rate(decim)), 1.0) * (2 * math.pi)
        wide += y * torch.complex(torch.cos(phase).float(), torch.sin(phase).float())
        del X, Y, y, phase
    del t
    g = torch.Generator(device="cuda")
    g.manual_seed(12 + decim)
    iq = torch.stack([wide.real, wide.imag], -1) + torch.randn((N, 2), generator=g, device="cuda") * 2.0
    x = torch.clamp(torch.round(iq), -32768, 32767).to(torch.int16).reshape(-1)
    return x[: x.numel() & ~63].cpu().numpy(), caps


@pytest.fixture(scope="module", params=DS)
def band(request):
    """The capture, the one-shot channeliser's output and the records of the one-shot path (nrsc5b_chan_run_device_cs16
    on the whole capture, the engine attached to its output, one nrsc5b_process)."""
    import torch
    import nrsc5_b200
    decim = request.param
    offs = [m for m, _, _, _ in STATIONS[decim]]
    x, caps = _band_capture(decim)
    d_x = torch.from_numpy(x).cuda()
    nout = ch.outputs(x.size, decim=decim)
    stride = (2 * nout + 64) & ~31
    d_out = torch.zeros((len(offs), stride), dtype=torch.int16, device="cuda")
    with ch.Channelizer(offs, input_cs16=True, decim=decim) as c:
        c.run_device(d_x.data_ptr(), x.size, d_out.data_ptr(), stride)
        torch.cuda.synchronize()
    with nrsc5_b200.Engine(nstreams=len(offs), input_capacity=4096, log_capacity=4 << 20, input_cs16=True) as e:
        e.attach_device_input(d_out.data_ptr(), 2 * stride, 4 * nout)
        e.process()
        recs = [e.drain(s) for s in range(len(offs))]
    return decim, offs, x, caps, d_out[:, : 2 * nout].cpu().numpy(), recs


@pytest.mark.gpu
def test_stations_decode_to_the_generator_and_the_oracle(band):
    import port
    from nrsc5_b200 import engine as eng, synth
    decim, offs, x, caps, y, recs = band
    assert np.abs(x).max() > 20000
    taps, ph = ch.make_tables(offs, decim=decim)
    assert np.array_equal(y[:, : 2 * 3000], rates.channelize(x[: 2 * (decim * 2999 + 256)], offs, taps, ph, decim))
    for s in range(len(offs)):
        p1 = [r["bits"] for t_, r in recs[s] if t_ == eng.REC_FRAME and r["lc"] == 0]
        assert any(synth.pack_bits(f) in p1 for f in caps[s].p1_frames), f"station {s}: its P1 PDU did not come out"
        ref = port.decode(y[s])
        assert p1 == ref.p1_frames, f"station {s}: P1 PDUs differ from the oracle's decode"
        assert [r["bits"] for t_, r in recs[s] if t_ == eng.REC_PIDS] == ref.pids_frames


def _without_positions(recs):
    """REC_BLOCK carries the block's start in the stream's input buffer, which a trim moves; everything else must agree."""
    from nrsc5_b200 import engine as eng
    return [(t, {k: v for k, v in r.items() if not (t == eng.REC_BLOCK and k == "start")}) for t, r in recs]


def _ragged(nvalues, seed):
    rng = np.random.default_rng(seed)
    cuts, pos = [0], 0
    while pos < nvalues:
        pos = min(nvalues, pos + (2 * int(rng.integers(1, 300)) if rng.random() < 0.2 else 2 * int(rng.integers(1 << 18, 3 << 19))))
        cuts.append(pos)
    return list(zip(cuts[:-1], cuts[1:]))


@pytest.mark.gpu
def test_feed_with_permuted_streams(band):
    import nrsc5_b200
    decim, offs, x, caps, _, ref = band
    nout = ch.outputs(x.size, decim=decim)
    perm = [2, 0, 1]
    with ch.Channelizer(offs, input_cs16=True, decim=decim) as c, \
            nrsc5_b200.Engine(nstreams=3, input_capacity=4 * nout + 4096, log_capacity=4 << 20, input_cs16=True) as e:
        for a, b in _ragged(x.size, 1):
            c.feed(e, x[a:b], streams=perm)
            e.process()
        got = [e.drain(perm[k]) for k in range(3)]
    assert got == ref


@pytest.mark.gpu
def test_feed_into_small_input_buffers_trims(band):
    import nrsc5_b200
    decim, offs, x, caps, _, ref = band
    cap = 3 << 20
    assert 4 * ch.outputs(x.size, decim=decim) > cap
    recs = [[] for _ in offs]
    with ch.Channelizer(offs, input_cs16=True, decim=decim) as c, \
            nrsc5_b200.Engine(nstreams=3, input_capacity=cap, log_capacity=4 << 20, input_cs16=True) as e:
        for a, b in _ragged(x.size, 2):
            c.feed(e, x[a:b])
            e.process()
            for s in range(3):
                recs[s] += e.drain(s)
    assert [_without_positions(r) for r in recs] == [_without_positions(r) for r in ref]


@pytest.mark.gpu
def test_feed_back_pressure_is_all_or_nothing(band):
    """Pushes without processing until the engine is full: the push that gets NRSC5B_EFULL takes nothing, neither in
    the channeliser nor in the engine, and the same values go in after nrsc5b_process."""
    import torch
    import nrsc5_b200
    decim, offs, x, caps, _, ref = band
    host = torch.from_numpy(x).pin_memory()
    step = (2 << 20) * decim // 32                                # int16 values per push: the same outputs at every D
    recs, refused = [[] for _ in offs], 0
    with ch.Channelizer(offs, input_cs16=True, decim=decim) as c, \
            nrsc5_b200.Engine(nstreams=3, input_capacity=1 << 20, log_capacity=4 << 20, input_cs16=True) as e:
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
                for s in range(3):
                    recs[s] += e.drain(s)
                c.feed(e, (host.data_ptr() + 2 * pos, n))
            pos += n
            if processing:
                e.process()
                for s in range(3):
                    recs[s] += e.drain(s)
        e.process()
        for s in range(3):
            recs[s] += e.drain(s)
        torch.cuda.synchronize()
    assert refused == 1
    assert [_without_positions(r) for r in recs] == [_without_positions(r) for r in ref]
