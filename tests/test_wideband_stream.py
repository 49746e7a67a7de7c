"""Streaming wideband ingest (include/nrsc5_b200.h: nrsc5b_chan_push / nrsc5b_chan_feed).  CPU tier: the streaming
definition restated here in numpy (channelize_stream, on top of oracle/chan_oracle.py's one-shot definition) against the
one-shot definition over random splits, and N(T) / the carry against their closed form.  GPU tier: the streamed kernel
bit for bit against the one-shot kernel and the definition, reset, the feed straight into a running cs16 engine
(permuted streams, trims, back-pressure) against the one-shot channeliser + engine path, and the feed's argument checks.  The channeliser runs on TMA and wgmma, which the CPU
emulation of the kernels does not model: there is no emulated twin."""
import numpy as np
import pytest

import chan_oracle
from nrsc5_b200 import channelizer as ch
from nrsc5_b200.engine import EngineError

WIDE = ch.WIDE_RATE
PERIOD = ch.PERIOD
DECIM = ch.DECIM


def stream_outputs(samples: int) -> int:
    """N(T): outputs whose 256-sample windows lie within the first T complex samples of a capture."""
    return (samples - ch.TAPS) // DECIM + 1 if samples >= ch.TAPS else 0


def channelize_stream(chunks, offsets, taps: np.ndarray, phasor: np.ndarray):
    """The streaming definition (include/nrsc5_b200.h, nrsc5b_chan_push): the capture arrives as `chunks` (uint8,
    each of even length, any of them empty).  A handle keeps T, the samples pushed so far, and the carry, the samples
    from 32 N(T) on; a push taking T to T' emits outputs N(T) .. N(T') - 1, computed from carry + chunk with the mixer
    at the absolute index n0 = N(T), and keeps the samples from 32 N(T') on.  Returns one int16 [nch][2 * n] array per
    push."""
    carry = np.zeros(0, dtype=np.uint8)
    pushed = 0
    outs = []
    for chunk in chunks:
        c = np.asarray(chunk, dtype=np.uint8).reshape(-1)
        assert c.size % 2 == 0, "pushes are whole complex samples"
        first, last = stream_outputs(pushed), stream_outputs(pushed + c.size // 2)
        held = np.concatenate([carry, c])                                      # starts at sample 32 N(T)
        n = last - first
        y = chan_oracle.channelize(held[: 64 * (n + 7)] if n > 0 else held[:0], offsets, taps, phasor, n0=first)
        assert y.shape[1] == 2 * n
        outs.append(y)
        pushed += c.size // 2
        carry = held[64 * n:]
        assert carry.size == 2 * (pushed - DECIM * last) <= 510
    return outs


def _splits(nbytes, rng, must=(), avoid=None):
    """Cut points of a capture into pushes of every awkward kind: empty, 2 bytes, shorter than the filter's 510 bytes,
    not a multiple of 64, large; plus the cuts in `must`, and none strictly inside the byte range `avoid`."""
    cuts, pos, i = [0], 0, 0
    while pos < nbytes:
        kind = i % 5
        if kind == 0:
            step = 0
        elif kind == 1:
            step = 2
        elif kind == 2:
            step = 2 * int(rng.integers(1, 255))
        elif kind == 3:
            step = 64 * int(rng.integers(1, 40)) + 2 * int(rng.integers(1, 32))
        else:
            step = 2 * int(rng.integers(20000, 200000))
        pos = min(nbytes, pos + step)
        cuts.append(pos)
        i += 1
    if avoid:
        cuts = [x for x in cuts if not avoid[0] < x < avoid[1]]
    cuts += [int(m) for m in must if 0 < m < nbytes]
    cuts.sort()
    return list(zip(cuts[:-1], cuts[1:]))


def _at_output(n):
    """The byte at which the capture holds exactly enough samples for outputs 0 .. n - 1."""
    return 2 * (32 * (n - 1) + 256)


# ---------------------------------------------------------------- CPU tier

def test_outputs_and_carry_closed_form():
    for t in list(range(0, 2000)) + [10 ** 6 + k for k in range(70)]:
        n = stream_outputs(t)
        assert n == sum(1 for m in range(t // 32 + 1) if 32 * m + 256 <= t)      # windows within the first t samples
        carry = t - 32 * n
        assert 0 <= carry <= 255 and (t < 256 or carry >= 224)
        assert n == ch.stream_outputs(0, 2 * t) == ch.outputs(2 * t)               # the binding's count, and the one-shot count
    assert ch.stream_outputs(300, 0) == 0 and ch.stream_outputs(255, 2) == 1 and ch.stream_outputs(256, 62) == 0


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_streamed_definition_equals_one_shot(seed):
    rng = np.random.default_rng(seed)
    offs = [int(m) for m in rng.choice(np.arange(-118, 119), 3, replace=False)]
    taps, ph = ch.make_tables(offs)
    nbytes = 2 * int(rng.integers(150000, 260000))
    cu8 = rng.integers(0, 256, nbytes, dtype=np.uint8)
    parts = _splits(nbytes, rng)
    assert any(b == a for a, b in parts) and any(b - a == 2 for a, b in parts) and any((b - a) % 64 for a, b in parts)
    outs = channelize_stream([cu8[a:b] for a, b in parts], offs, taps, ph)
    want = chan_oracle.channelize(cu8, offs, taps, ph)
    assert [o.shape[1] for o in outs] == [2 * ch.stream_outputs(a // 2, b - a) for a, b in parts]
    assert np.array_equal(np.concatenate(outs, axis=1), want)


# ---------------------------------------------------------------- GPU tier

@pytest.mark.gpu
@pytest.mark.parametrize("nch", [3, 40, 33])
def test_streamed_kernel_equals_one_shot_bit_for_bit(nch):
    """Random splits, the mixer wrapping inside a push (output 11907) and at a push boundary (output 2 x 11907)."""
    import torch
    rng = np.random.default_rng(100 + nch)
    offs = list(rng.choice(np.arange(-118, 119), nch, replace=False))
    nbytes = 64 * 25001 + 38
    cu8 = rng.integers(0, 256, nbytes, dtype=np.uint8)
    lo, hi = _at_output(PERIOD) - 64 * 500, _at_output(PERIOD) + 64 * 500
    parts = _splits(nbytes, rng, must=[_at_output(2 * PERIOD), lo, hi], avoid=(lo, hi))
    assert (lo, hi) in parts                                    # one push emits outputs 11407 .. 12406: the wrap inside it
    assert any(b == _at_output(2 * PERIOD) for a, b in parts)   # the next push starts at output 2 x 11907
    with ch.Channelizer(offs) as c:
        taps, ph = c.tables()
        whole = c.run(cu8)
        got = [c.push(cu8[a:b]) for a, b in parts]
        assert c.pushed == nbytes // 2
        # the same through push_device, with the capture in device memory and in page-locked host memory
        c.reset()
        d_cu8 = torch.from_numpy(cu8).cuda()
        h_cu8 = torch.from_numpy(cu8).pin_memory()
        nout = ch.outputs(nbytes)
        d_out = torch.zeros((nch, 2 * nout + 64), dtype=torch.int16, device="cuda")
        col = 0
        for i, (a, b) in enumerate(parts):
            src = d_cu8 if i % 2 else h_cu8
            n = c.push_device(src.data_ptr() + a, b - a, d_out.data_ptr() + 2 * col, d_out.shape[1])
            col += 2 * n
        torch.cuda.synchronize()
        assert col == 2 * nout
    want = chan_oracle.channelize(cu8, offs, taps, ph)
    assert np.array_equal(whole, want)
    assert [g.shape[1] for g in got] == [2 * ch.stream_outputs(a // 2, b - a) for a, b in parts]
    cat = np.concatenate(got, axis=1)
    bad = np.argwhere(cat != want)
    assert bad.size == 0, f"{bad.shape[0]} of {cat.size} values differ; first at (channel, value) {bad[:5].tolist()}"
    assert np.array_equal(d_out[:, : 2 * nout].cpu().numpy(), want)


@pytest.mark.gpu
def test_push_larger_than_the_staging_buffer():
    """A push of 9 MiB goes through the 4 MiB staging buffer in pieces; the outputs are the one-shot kernel's."""
    rng = np.random.default_rng(9)
    offs = [0, 31, -77, 50, -118]
    nbytes = (9 << 20) + 6
    cu8 = rng.integers(0, 256, nbytes, dtype=np.uint8)
    with ch.Channelizer(offs) as c:
        taps, ph = c.tables()
        whole = c.run(cu8)
        got = np.concatenate([c.push(cu8[:302]), c.push(cu8[302: nbytes - 1000]), c.push(cu8[nbytes - 1000:])], axis=1)
    assert np.array_equal(got, whole)
    nout = ch.outputs(nbytes)
    tail = chan_oracle.channelize(cu8[64 * (nout - 300):], offs, taps, ph, n0=nout - 300)
    assert np.array_equal(got[:, 2 * (nout - 300):], tail)


@pytest.mark.gpu
def test_reset_starts_the_stream_over():
    rng = np.random.default_rng(4)
    offs = [12, -3, 99]
    cu8 = rng.integers(0, 256, 64 * 3000 + 10, dtype=np.uint8)
    with ch.Channelizer(offs) as fresh:
        want = np.concatenate([fresh.push(cu8[:5000]), fresh.push(cu8[5000:])], axis=1)
    with ch.Channelizer(offs) as c:
        c.push(rng.integers(0, 256, 64 * 777 + 130, dtype=np.uint8))   # leaves a carry and a mixer position behind
        c.reset()
        assert c.pushed == 0
        got = np.concatenate([c.push(cu8[:5000]), c.push(cu8[5000:])], axis=1)
    assert np.array_equal(got, want)


# ---- the feed straight into a running engine

OFFS = [11, -23]


def _two_station_capture():
    """Two synthetic FM MP1 stations 1.1 MHz and -2.3 MHz from the capture centre, plus noise, at 23.814 MS/s cu8: the
    capture of test_channelizer.py::test_stations_in_a_wideband_capture_decode_bit_exact, rebuilt the same way."""
    import scipy.fft
    from nrsc5_b200 import synth
    caps = [synth.make_fm_mp1(nframes=1, seed=70 + i, lead_in=900 * i + 40, tail_blocks=3) for i in range(2)]
    n = min(c.cu8.size for c in caps) // 2
    up = 16
    wide = np.zeros(n * up, dtype=np.complex64)
    t = np.arange(n * up, dtype=np.float64)
    for c, m in zip(caps, OFFS):
        x = (c.cu8[0:2 * n:2].astype(np.float32) - 127) + 1j * (c.cu8[1:2 * n:2].astype(np.float32) - 127)
        X = scipy.fft.fft(x.astype(np.complex64))
        Y = np.zeros(n * up, dtype=np.complex64)                          # band-limited interpolation by 16
        Y[: n // 2] = X[: n // 2]
        Y[-(n - n // 2):] = X[n // 2:]
        y = scipy.fft.ifft(Y) * up
        wide += (y * np.exp(2j * np.pi * (m * 100e3 / WIDE) * t)).astype(np.complex64)
    rng = np.random.default_rng(5)
    wide += (rng.standard_normal(wide.size) + 1j * rng.standard_normal(wide.size)).astype(np.complex64) * 2.0
    cu8 = np.empty(2 * wide.size, dtype=np.uint8)
    cu8[0::2] = np.clip(np.rint(wide.real + 127), 0, 255)
    cu8[1::2] = np.clip(np.rint(wide.imag + 127), 0, 255)
    return cu8[: cu8.size & ~63], caps


@pytest.fixture(scope="module")
def two_stations():
    """The capture and the records of the one-shot path: nrsc5b_chan_run_device on the whole capture, the engine
    attached to its output, one nrsc5b_process."""
    import torch
    import nrsc5_b200
    cu8, caps = _two_station_capture()
    d_cu8 = torch.from_numpy(cu8).cuda()
    nout = ch.outputs(cu8.size)
    stride = (2 * nout + 64) & ~31
    d_out = torch.zeros((2, stride), dtype=torch.int16, device="cuda")
    with ch.Channelizer(OFFS) as c:
        c.run_device(d_cu8.data_ptr(), cu8.size, d_out.data_ptr(), stride)
        torch.cuda.synchronize()
    with nrsc5_b200.Engine(nstreams=2, input_capacity=4096, log_capacity=4 << 20, input_cs16=True) as e:
        e.attach_device_input(d_out.data_ptr(), 2 * stride, 4 * nout)
        e.process()
        recs = [e.drain(s) for s in range(2)]
    return cu8, caps, recs


def _ragged(nbytes, seed):
    rng = np.random.default_rng(seed)
    cuts, pos = [0], 0
    while pos < nbytes:
        pos = min(nbytes, pos + (2 * int(rng.integers(1, 300)) if rng.random() < 0.2 else 2 * int(rng.integers(1 << 19, 3 << 20))))
        cuts.append(pos)
    return list(zip(cuts[:-1], cuts[1:]))


def _without_positions(recs):
    """REC_BLOCK carries the block's start in the stream's input buffer, which a trim moves; everything else must agree."""
    from nrsc5_b200 import engine as eng
    return [(t, {k: v for k, v in r.items() if not (t == eng.REC_BLOCK and k == "start")}) for t, r in recs]


def _check_stations(recs, caps, ref):
    from nrsc5_b200 import engine as eng, synth
    for s in range(2):
        p1 = [r["bits"] for t_, r in recs[s] if t_ == eng.REC_FRAME and r["lc"] == 0]
        assert any(synth.pack_bits(f) in p1 for f in caps[s].p1_frames), f"station {s}: its P1 PDU did not come out"
        assert recs[s] == ref[s]


@pytest.mark.gpu
def test_feed_with_permuted_streams(two_stations):
    import nrsc5_b200
    cu8, caps, ref = two_stations
    nout = ch.outputs(cu8.size)
    with ch.Channelizer(OFFS) as c, nrsc5_b200.Engine(nstreams=2, input_capacity=4 * nout + 4096, log_capacity=4 << 20,
                                                      input_cs16=True) as e:
        for a, b in _ragged(cu8.size, 1):
            c.feed(e, cu8[a:b], streams=[1, 0])                          # channel 0 -> stream 1, channel 1 -> stream 0
            e.process()
        got = [e.drain(1), e.drain(0)]
    _check_stations(got, caps, ref)


@pytest.mark.gpu
def test_feed_into_small_input_buffers_trims(two_stations):
    import nrsc5_b200
    cu8, caps, ref = two_stations
    cap = 3 << 20                                                       # well below the 5 MB each station's cs16 takes
    assert 4 * ch.outputs(cu8.size) > cap
    recs = [[], []]
    with ch.Channelizer(OFFS) as c, nrsc5_b200.Engine(nstreams=2, input_capacity=cap, log_capacity=4 << 20, input_cs16=True) as e:
        for a, b in _ragged(cu8.size, 2):
            c.feed(e, cu8[a:b])
            e.process()
            for s in range(2):
                recs[s] += e.drain(s)
    assert [_without_positions(r) for r in recs] == [_without_positions(r) for r in ref]
    _check_stations([_without_positions(r) for r in recs], caps, [_without_positions(r) for r in ref])


@pytest.mark.gpu
def test_feed_back_pressure_is_all_or_nothing(two_stations):
    """Pushes without processing until the engine is full: the push that gets NRSC5B_EFULL takes nothing, neither in
    the channeliser nor in the engine, and the same bytes go in after nrsc5b_process."""
    import torch
    import nrsc5_b200
    cu8, caps, ref = two_stations
    host = torch.from_numpy(cu8).pin_memory()                           # page-locked input, as a live source would hand it over
    step = 2 << 20
    recs, refused = [[], []], 0
    with ch.Channelizer(OFFS) as c, nrsc5_b200.Engine(nstreams=2, input_capacity=1 << 20, log_capacity=4 << 20,
                                                      input_cs16=True) as e:
        pos, processing = 0, False
        while pos < cu8.size:
            n = min(step, cu8.size - pos)
            before = c.pushed
            try:
                c.feed(e, (host.data_ptr() + pos, n))
            except EngineError as ex:
                assert "EFULL" in str(ex) and not processing
                assert c.pushed == before
                refused += 1
                processing = True                                       # from now on: process after every push
                e.process()
                for s in range(2):
                    recs[s] += e.drain(s)
                c.feed(e, (host.data_ptr() + pos, n))                   # the same bytes again
            pos += n
            if processing:
                e.process()
                for s in range(2):
                    recs[s] += e.drain(s)
        e.process()
        for s in range(2):
            recs[s] += e.drain(s)
        torch.cuda.synchronize()
    assert refused == 1
    _check_stations([_without_positions(r) for r in recs], caps, [_without_positions(r) for r in ref])


@pytest.mark.gpu
def test_feed_argument_checks_change_nothing():
    import nrsc5_b200
    rng = np.random.default_rng(3)
    offs = [5, -60]
    cu8 = rng.integers(0, 256, 64 * 2000 + 14, dtype=np.uint8)
    with ch.Channelizer(offs) as want_c:
        want = np.concatenate([want_c.push(cu8[:1000]), want_c.push(cu8[1000:])], axis=1)
    with ch.Channelizer(offs) as c:
        first = c.push(cu8[:1000])
        with nrsc5_b200.Engine(nstreams=2, input_capacity=1 << 16, mode="am", input_cs16=True) as am, \
                nrsc5_b200.Engine(nstreams=2, input_capacity=1 << 16, input_cs16=False) as fm_cu8, \
                nrsc5_b200.Engine(nstreams=3, input_capacity=1 << 20, log_capacity=1 << 16, input_cs16=True) as e:
            bad = [(am, None, cu8[1000:]), (fm_cu8, None, cu8[1000:]), (e, [1, 1], cu8[1000:]), (e, [0, 3], cu8[1000:]),
                   (e, [-1, 0], cu8[1000:]), (e, None, cu8[1000:1001])]
            for eng_, streams, data in bad:
                with pytest.raises(EngineError, match="EINVAL"):
                    c.feed(eng_, data, streams=streams)
                assert c.pushed == 500
            with ch.Channelizer([0, 1, 2, 3]) as wide:                 # more channels than the engine has streams
                with pytest.raises(EngineError, match="EINVAL"):
                    wide.feed(e, cu8)
            # a valid feed then continues the stream where the first push left it
            c.feed(e, cu8[1000:60000], streams=[2, 0])
            e.process()
        assert c.pushed == 30000
        assert c.push(np.zeros(0, dtype=np.uint8)).shape == (2, 0)
        rest = c.push(cu8[60000:])
    assert np.array_equal(first, want[:, : first.shape[1]])
    assert np.array_equal(rest, want[:, 2 * stream_outputs(30000):])
