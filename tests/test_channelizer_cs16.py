"""The wideband channeliser on cs16 input (include/nrsc5_b200.h: nrsc5b_chan_*_cs16).  CPU tier: the numpy
definition (tests/chan_oracle_cs16.py) against the cu8 definition on 64 (cu8 - 127), the saturation of v on
full-scale input, and the streamed restatement against the one-shot one.  GPU tier: the kernel against the definition
bit for bit, against the cu8 kernel on scaled input, streamed against one-shot, the feed into a running cs16 engine
against the one-shot channeliser + engine path, and stations 48 dB apart in one 16-bit capture all decoding.  The
channeliser runs on TMA and wgmma, which the CPU emulation of the kernels does not model: there is no emulated twin."""
import ctypes

import numpy as np
import pytest

import chan_oracle
import chan_oracle_cs16
from nrsc5_b200 import channelizer as ch
from nrsc5_b200.engine import EngineError

WIDE = ch.WIDE_RATE
PERIOD = ch.PERIOD
DECIM = ch.DECIM
EINVAL = -2


def _offsets(rng, nch):
    """nch distinct channel offsets spread over the whole +-118 range (both ends included)."""
    inner = [int(m) for m in rng.choice(np.arange(-117, 118), nch - 2, replace=False)]
    return [-118] + inner + [118]


def _full_range(rng, nvalues):
    x = rng.integers(-32768, 32768, nvalues, dtype=np.int16)
    x[rng.integers(0, nvalues, 64)] = -32768
    x[rng.integers(0, nvalues, 64)] = 32767
    return x


def _saturating_window(taps, k):
    """256 samples of +-32767 in the sign pattern of channel k's taps (real part of acc maximal): xr = sgn(Wr),
    xi = -sgn(Wi), so Re(acc) = 32767 sum(|Wr| + |Wi|) ~ 1.4 x 2^19 x 32767 and v would be ~ 1.4 x 32767."""
    wr, wi = taps[k, :, 0].astype(np.int64), taps[k, :, 1].astype(np.int64)
    x = np.empty(2 * ch.TAPS, dtype=np.int16)
    x[0::2] = np.where(wr >= 0, 32767, -32767)
    x[1::2] = np.where(wi >= 0, -32767, 32767)
    return x


def _v_unsaturated(cs16, taps, k, n):
    """The real part of v before sat16 for output n of channel k."""
    x = cs16.astype(np.int64)
    xr, xi = x[0::2][DECIM * n: DECIM * n + ch.TAPS], x[1::2][DECIM * n: DECIM * n + ch.TAPS]
    acc = int(xr @ taps[k, :, 0].astype(np.int64) - xi @ taps[k, :, 1].astype(np.int64))
    return (acc + (1 << 18)) >> 19


def _splits(nvalues, rng, big=(20000, 200000)):
    """Cut points (in int16 values) of a capture into pushes of every awkward kind: empty, one sample, fewer than 256
    samples, not a multiple of 32 samples, large."""
    cuts, pos, i = [0], 0, 0
    while pos < nvalues:
        kind = i % 5
        step = [0, 2, 2 * int(rng.integers(1, 256)), 64 * int(rng.integers(1, 40)) + 2 * int(rng.integers(1, 32)),
                2 * int(rng.integers(*big))][kind]
        pos = min(nvalues, pos + step)
        cuts.append(pos)
        i += 1
    return list(zip(cuts[:-1], cuts[1:]))


# ---------------------------------------------------------------- CPU tier

@pytest.mark.parametrize("seed", [1, 2])
def test_cs16_definition_is_the_cu8_definition_on_scaled_input(seed):
    rng = np.random.default_rng(seed)
    offs = _offsets(rng, 4)
    taps, ph = ch.make_tables(offs)
    cu8 = rng.integers(0, 256, 64 * 900, dtype=np.uint8)
    cu8[:64] = 0                                                 # the extremes of the cu8 range as well
    cu8[64:128] = 255
    x16 = (64 * (cu8.astype(np.int16) - 127)).astype(np.int16)
    assert np.array_equal(chan_oracle_cs16.channelize_cs16(x16, offs, taps, ph), chan_oracle.channelize(cu8, offs, taps, ph))
    assert np.array_equal(chan_oracle_cs16.channelize_cs16(x16[: 2 * 5000], offs, taps, ph, n0=11900),
                          chan_oracle.channelize(cu8[: 2 * 5000 & ~63], offs, taps, ph, n0=11900)[:, : 2 * ((5000 - 256) // 32 + 1)])


def test_cs16_v_saturates_on_full_scale_input():
    offs = [0, 37, -101]
    taps, ph = ch.make_tables(offs)
    rng = np.random.default_rng(8)
    for k in range(len(offs)):
        x = np.concatenate([_saturating_window(taps, k), _full_range(rng, 2 * 32 * 40)])
        v = _v_unsaturated(x, taps, k, 0)
        assert v > 40000                                          # beyond int16: sat16 is what the rotation sees
        y = chan_oracle_cs16.channelize_cs16(x, offs, taps, ph)
        # output 0 by hand: the phasor index is 0, conj(P[0]) = 32767, so y = (sat16(v) * 32767 + 2^14) >> 15 per part
        xr, xi = x[0:512:2].astype(np.int64), x[1:512:2].astype(np.int64)
        vi = (int(xi @ taps[k, :, 0].astype(np.int64) + xr @ taps[k, :, 1].astype(np.int64)) + (1 << 18)) >> 19
        vi = min(32767, max(-32768, vi))
        assert ph[0, 0] == 32767 and ph[0, 1] == 0
        assert y[k, 0] == (32767 * 32767 + (1 << 14)) >> 15 == 32766   # without sat16 on v it would clamp at 32767
        assert y[k, 1] == (vi * 32767 + (1 << 14)) >> 15


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_cs16_streamed_definition_equals_one_shot(seed):
    rng = np.random.default_rng(seed)
    offs = _offsets(rng, 3)
    taps, ph = ch.make_tables(offs)
    nvalues = 2 * int(rng.integers(150000, 260000))
    x = _full_range(rng, nvalues)
    parts = _splits(nvalues, rng)
    sizes = [b - a for a, b in parts]
    assert 0 in sizes and 2 in sizes and any(0 < s < 512 for s in sizes) and any((s // 2) % 32 for s in sizes)
    outs = chan_oracle_cs16.channelize_cs16_stream([x[a:b] for a, b in parts], offs, taps, ph)
    assert [o.shape[1] for o in outs] == [2 * ch.stream_outputs(a // 2, b - a) for a, b in parts]
    assert np.array_equal(np.concatenate(outs, axis=1), chan_oracle_cs16.channelize_cs16(x, offs, taps, ph))


def test_cs16_channelizer_needs_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(EngineError):
        ch.Channelizer([0, 9], input_cs16=True)


# ---------------------------------------------------------------- GPU tier

@pytest.mark.gpu
@pytest.mark.parametrize("nch,nsamples", [(3, 32 * 700), (40, 32 * 1031 + 5), (33, 32 * 135 + 1), (5, 32 * 12100 + 17)])
def test_cs16_kernel_equals_the_definition_bit_for_bit(nch, nsamples):
    """Random full-range input with a saturating window at the front of every channel's first outputs; 33 / 40
    channels leave a partial last group; the last case runs past output 11907, where the mixer wraps."""
    rng = np.random.default_rng(50 + nch)
    offs = _offsets(rng, nch)
    with ch.Channelizer(offs, input_cs16=True) as c:
        taps, ph = c.tables()
        t2, p2 = ch.make_tables(offs)
        assert np.array_equal(taps, t2) and np.array_equal(ph, p2)
        x = _full_range(rng, 2 * nsamples)
        for j, k in enumerate(range(0, nch, max(1, nch // 4))):  # saturating windows for outputs 0, 8, 16, ...
            x[2 * 256 * j: 2 * 256 * (j + 1)] = _saturating_window(taps, k)
            assert abs(_v_unsaturated(x, taps, k, 8 * j)) > 32767
        got = c.run(x)
    want = chan_oracle_cs16.channelize_cs16(x, offs, taps, ph)
    assert got.shape == want.shape == (nch, 2 * ((nsamples - 256) // 32 + 1))
    bad = np.argwhere(got != want)
    assert bad.size == 0, f"{bad.shape[0]} of {got.size} values differ; first at (channel, value) {bad[:5].tolist()}: " \
                          f"got {got[tuple(bad[0])]} want {want[tuple(bad[0])]}"


@pytest.mark.gpu
def test_cs16_kernel_on_scaled_cu8_equals_the_cu8_kernel():
    """x16 = 64 (x8 - 127): the cs16 kernel's output is the cu8 kernel's, one-shot and streamed."""
    rng = np.random.default_rng(21)
    offs = _offsets(rng, 35)
    cu8 = rng.integers(0, 256, 64 * 20000, dtype=np.uint8)
    x16 = (64 * (cu8.astype(np.int16) - 127)).astype(np.int16)
    parts = _splits(x16.size, rng)
    with ch.Channelizer(offs) as c8, ch.Channelizer(offs, input_cs16=True) as c16:
        want = c8.run(cu8)
        assert np.array_equal(c16.run(x16), want)
        s8 = np.concatenate([c8.push(cu8[a:b]) for a, b in parts], axis=1)
        s16 = np.concatenate([c16.push(x16[a:b]) for a, b in parts], axis=1)
    assert np.array_equal(s8, want) and np.array_equal(s16, want)


@pytest.mark.gpu
@pytest.mark.parametrize("nch", [3, 33])
def test_cs16_streamed_equals_one_shot_from_every_kind_of_memory(nch):
    """Awkward splits, from pageable, page-locked and device memory, the mixer wrapping inside the stream; then reset
    and the same again."""
    import torch
    rng = np.random.default_rng(200 + nch)
    offs = _offsets(rng, nch)
    nvalues = 2 * (32 * 25001 + 19)
    x = _full_range(rng, nvalues)
    parts = _splits(nvalues, rng)
    nout = ch.outputs(nvalues)
    d_x = torch.from_numpy(x).cuda()
    h_x = torch.from_numpy(x).pin_memory()
    with ch.Channelizer(offs, input_cs16=True) as c:
        taps, ph = c.tables()
        whole = c.run(x)
        for rep in range(2):                                     # the second time after a reset
            if rep:
                c.reset()
                assert c.pushed == 0
            got = []
            d_out = torch.zeros((nch, 2 * nout + 64), dtype=torch.int16, device="cuda")
            col = 0
            for i, (a, b) in enumerate(parts):
                if i % 3 == 0:
                    got.append(c.push(x[a:b]))                    # pageable
                    d_out[:, col: col + got[-1].shape[1]] = torch.from_numpy(got[-1]).cuda()
                    col += got[-1].shape[1]
                else:
                    src = d_x if i % 3 == 1 else h_x
                    n = c.push_device(src.data_ptr() + 2 * a, b - a, d_out.data_ptr() + 2 * col, d_out.shape[1])
                    col += 2 * n
            torch.cuda.synchronize()
            assert col == 2 * nout and c.pushed == nvalues // 2
            streamed = d_out[:, : 2 * nout].cpu().numpy()
            bad = np.argwhere(streamed != whole)
            assert bad.size == 0, f"pass {rep}: {bad.shape[0]} values differ; first at {bad[:5].tolist()}"
    assert np.array_equal(whole, chan_oracle_cs16.channelize_cs16(x, offs, taps, ph))


@pytest.mark.gpu
def test_cs16_capture_larger_than_the_scratch():
    """A capture of 2^22 + 300 000 samples: the one-shot device entry goes through the 2^22-sample planes in two
    pieces and leaves its input unchanged; one push larger than the staging buffer goes through it in pieces.  Both
    equal the definition at the start, across the piece boundary (output 2^17) and at the end."""
    import torch
    rng = np.random.default_rng(31)
    offs = [0, 31, -77, 50, -118, 118]
    nvalues = 2 * ((1 << 22) + 300000)
    x = _full_range(rng, nvalues)
    nout = ch.outputs(nvalues)
    stride = 2 * nout + 32
    d_x = torch.from_numpy(x).cuda()
    before = d_x.clone()
    with ch.Channelizer(offs, input_cs16=True) as c:
        taps, ph = c.tables()
        d_out = torch.zeros((len(offs), stride), dtype=torch.int16, device="cuda")
        c.run_device(d_x.data_ptr(), nvalues, d_out.data_ptr(), stride)
        torch.cuda.synchronize()
        assert torch.equal(d_x, before), "the one-shot entry wrote to its input"
        one = d_out[:, : 2 * nout].cpu().numpy()
        got = np.concatenate([c.push(x[:302]), c.push(x[302: nvalues - 1000]), c.push(x[nvalues - 1000:])], axis=1)
    assert np.array_equal(got, one)
    for n0, n in ((0, 600), ((1 << 17) - 300, 600), (nout - 300, 300)):
        want = chan_oracle_cs16.channelize_cs16(x[2 * DECIM * n0: 2 * (DECIM * (n0 + n) + 224)], offs, taps, ph, n0=n0)
        assert np.array_equal(one[:, 2 * n0: 2 * (n0 + n)], want), f"outputs {n0} .. {n0 + n - 1}"


# ---- stations 48 dB apart in one 16-bit capture, and the feed straight into a running engine

OFFS = [11, -23, 40]                                             # 1.1, -2.3 and 4.0 MHz from the capture centre
SCALES = [250.0, 1.0, 16.0]                                      # x (cu8 - 127): 48 dB and 24 dB below the strong station


def _band(device="cuda"):
    """Three synthetic FM MP1 stations interpolated by 16 (band-limited, on the GPU) into one 23.814 MS/s cs16
    capture with a little noise: the strongest near full scale (rms 5000, peaks near 32767), the weakest 48 dB below
    it (rms 20 LSB, under one LSB of any 8-bit quantisation of the same band)."""
    import math
    import torch
    from nrsc5_b200 import synth
    caps = [synth.make_fm_mp1(nframes=1, seed=80 + i, lead_in=700 * i + 40, tail_blocks=3) for i in range(len(OFFS))]
    n = min(c.cu8.size for c in caps) // 2
    up = 16
    N = n * up
    wide = torch.zeros(N, dtype=torch.complex64, device=device)
    t = torch.arange(N, dtype=torch.float64, device=device)
    for c, m, s in zip(caps, OFFS, SCALES):
        xi = torch.from_numpy(c.cu8[: 2 * n].astype(np.float32) - 127.0).to(device).view(-1, 2)
        X = torch.fft.fft(torch.complex(xi[:, 0].contiguous(), xi[:, 1].contiguous()))
        Y = torch.zeros(N, dtype=torch.complex64, device=device)
        Y[: n // 2] = X[: n // 2]
        Y[-(n - n // 2):] = X[n // 2:]
        y = torch.fft.ifft(Y) * (up * s)
        ph = torch.remainder(t * (m * 100e3 / WIDE), 1.0) * (2 * math.pi)
        wide += y * torch.complex(torch.cos(ph).float(), torch.sin(ph).float())
        del X, Y, y, ph
    del t
    g = torch.Generator(device=device)
    g.manual_seed(12)
    iq = torch.stack([wide.real, wide.imag], -1) + torch.randn((N, 2), generator=g, device=device) * 2.0
    del wide
    x = torch.clamp(torch.round(iq), -32768, 32767).to(torch.int16).reshape(-1)
    nvalues = x.numel() & ~63
    return x[:nvalues].cpu().numpy(), caps


@pytest.fixture(scope="module")
def band():
    """The capture, the one-shot channeliser's output and the records of the one-shot path (nrsc5b_chan_run_device_cs16
    on the whole capture, the engine attached to its output, one nrsc5b_process)."""
    import torch
    import nrsc5_b200
    x, caps = _band()
    d_x = torch.from_numpy(x).cuda()
    nout = ch.outputs(x.size)
    stride = (2 * nout + 64) & ~31
    d_out = torch.zeros((len(OFFS), stride), dtype=torch.int16, device="cuda")
    with ch.Channelizer(OFFS, input_cs16=True) as c:
        c.run_device(d_x.data_ptr(), x.size, d_out.data_ptr(), stride)
        torch.cuda.synchronize()
    with nrsc5_b200.Engine(nstreams=len(OFFS), input_capacity=4096, log_capacity=4 << 20, input_cs16=True) as e:
        e.attach_device_input(d_out.data_ptr(), 2 * stride, 4 * nout)
        e.process()
        recs = [e.drain(s) for s in range(len(OFFS))]
    return x, caps, d_out[:, : 2 * nout].cpu().numpy(), recs


def _p1(recs):
    from nrsc5_b200 import engine as eng
    return [r["bits"] for t_, r in recs if t_ == eng.REC_FRAME and r["lc"] == 0]


@pytest.mark.gpu
def test_cs16_stations_48_db_apart_all_decode(band):
    """Every station's P1 PDUs include its generated frames and equal what the CPU oracle decodes from the
    channeliser's output for that channel; the start of that output is the definition's."""
    import port
    from nrsc5_b200 import synth
    x, caps, cs16, recs = band
    assert np.abs(x).max() > 20000                               # the strong station reaches near full scale
    taps, ph = ch.make_tables(OFFS)
    assert np.array_equal(cs16[:, : 2 * 3000], chan_oracle_cs16.channelize_cs16(x[: 2 * (32 * 3000 + 224)], OFFS, taps, ph))
    for s in range(len(OFFS)):
        p1 = _p1(recs[s])
        assert any(synth.pack_bits(f) in p1 for f in caps[s].p1_frames), f"station {s}: its P1 PDU did not come out"
        assert p1 == port.decode(cs16[s]).p1_frames, f"station {s}: P1 PDUs differ from the oracle's decode"


def _without_positions(recs):
    """REC_BLOCK carries the block's start in the stream's input buffer, which a trim moves; everything else must agree."""
    from nrsc5_b200 import engine as eng
    return [(t, {k: v for k, v in r.items() if not (t == eng.REC_BLOCK and k == "start")}) for t, r in recs]


def _ragged(nvalues, seed):
    rng = np.random.default_rng(seed)
    cuts, pos = [0], 0
    while pos < nvalues:
        pos = min(nvalues, pos + (2 * int(rng.integers(1, 300)) if rng.random() < 0.2 else 2 * int(rng.integers(1 << 19, 3 << 20))))
        cuts.append(pos)
    return list(zip(cuts[:-1], cuts[1:]))


@pytest.mark.gpu
def test_cs16_feed_with_permuted_streams(band):
    import nrsc5_b200
    x, caps, _, ref = band
    nout = ch.outputs(x.size)
    perm = [2, 0, 1]
    with ch.Channelizer(OFFS, input_cs16=True) as c, \
            nrsc5_b200.Engine(nstreams=3, input_capacity=4 * nout + 4096, log_capacity=4 << 20, input_cs16=True) as e:
        for a, b in _ragged(x.size, 1):
            c.feed(e, x[a:b], streams=perm)                      # channel k -> stream perm[k]
            e.process()
        got = [e.drain(perm[k]) for k in range(3)]
    assert got == ref


@pytest.mark.gpu
def test_cs16_feed_into_small_input_buffers_trims(band):
    import nrsc5_b200
    x, caps, _, ref = band
    cap = 3 << 20
    assert 4 * ch.outputs(x.size) > cap
    recs = [[], [], []]
    with ch.Channelizer(OFFS, input_cs16=True) as c, \
            nrsc5_b200.Engine(nstreams=3, input_capacity=cap, log_capacity=4 << 20, input_cs16=True) as e:
        for a, b in _ragged(x.size, 2):
            c.feed(e, x[a:b])
            e.process()
            for s in range(3):
                recs[s] += e.drain(s)
    assert [_without_positions(r) for r in recs] == [_without_positions(r) for r in ref]


@pytest.mark.gpu
def test_cs16_feed_back_pressure_is_all_or_nothing(band):
    """Pushes without processing until the engine is full: the push that gets NRSC5B_EFULL takes nothing, neither in
    the channeliser nor in the engine, and the same values go in after nrsc5b_process."""
    import torch
    import nrsc5_b200
    x, caps, _, ref = band
    host = torch.from_numpy(x).pin_memory()
    step = 2 << 20                                               # int16 values per push
    recs, refused = [[], [], []], 0
    with ch.Channelizer(OFFS, input_cs16=True) as c, \
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


@pytest.mark.gpu
def test_cs16_format_and_argument_checks_change_nothing():
    """cu8 entry points on a cs16 handle, cs16 ones on a cu8 handle, odd value counts, a misaligned device capture: all
    NRSC5B_EINVAL, and the stream goes on as if they had not been made."""
    import torch
    import nrsc5_b200
    rng = np.random.default_rng(3)
    offs = [5, -60]
    x = _full_range(rng, 64 * 2000 + 14)
    cu8 = rng.integers(0, 256, 64 * 2000 + 14, dtype=np.uint8)
    with ch.Channelizer(offs, input_cs16=True) as want16, ch.Channelizer(offs) as want8:
        w16 = np.concatenate([want16.push(x[:1000]), want16.push(x[1000:])], axis=1)
        w8 = np.concatenate([want8.push(cu8[:1000]), want8.push(cu8[1000:])], axis=1)
    L = ch._lib()
    vp = ctypes.c_void_p
    d_out = torch.zeros((2, 8192), dtype=torch.int16, device="cuda")
    d_in = torch.zeros(1 << 16, dtype=torch.int16, device="cuda")
    host_out = np.zeros((2, 8192), dtype=np.int16)
    nout = ctypes.c_longlong(7)
    with ch.Channelizer(offs, input_cs16=True) as c16, ch.Channelizer(offs) as c8, \
            nrsc5_b200.Engine(nstreams=3, input_capacity=1 << 20, log_capacity=1 << 16, input_cs16=True) as e:
        f16, f8 = c16.push(x[:1000]), c8.push(cu8[:1000])
        h16, h8 = c16._h, c8._h
        a16, a8 = x[1000:3000], cu8[1000:3000]
        calls = [
            L.nrsc5b_chan_push(h16, a8.ctypes.data, a8.size, vp(d_out.data_ptr()), 8192, None, ctypes.byref(nout)),
            L.nrsc5b_chan_feed(h16, e._h, None, a8.ctypes.data, a8.size),
            L.nrsc5b_chan_run(h16, a8.ctypes.data, a8.size, host_out.ctypes.data),
            L.nrsc5b_chan_run_device(h16, vp(d_in.data_ptr()), 4096, vp(d_out.data_ptr()), 8192, None),
            L.nrsc5b_chan_push_cs16(h8, a16.ctypes.data, a16.size, vp(d_out.data_ptr()), 8192, None, None),
            L.nrsc5b_chan_feed_cs16(h8, e._h, None, a16.ctypes.data, a16.size),
            L.nrsc5b_chan_run_cs16(h8, a16.ctypes.data, a16.size, host_out.ctypes.data),
            L.nrsc5b_chan_run_device_cs16(h8, vp(d_in.data_ptr()), 4096, vp(d_out.data_ptr()), 8192, None),
            L.nrsc5b_chan_push_cs16(h16, a16.ctypes.data, 1001, vp(d_out.data_ptr()), 8192, None, None),
            L.nrsc5b_chan_feed_cs16(h16, e._h, None, a16.ctypes.data, 1001),
            L.nrsc5b_chan_run_cs16(h16, a16.ctypes.data, 1001, host_out.ctypes.data),
            L.nrsc5b_chan_run_device_cs16(h16, vp(d_in.data_ptr()), 4097, vp(d_out.data_ptr()), 8192, None),
            L.nrsc5b_chan_run_device_cs16(h16, vp(d_in.data_ptr() + 8), 4096, vp(d_out.data_ptr()), 8192, None),
        ]
        assert calls == [EINVAL] * len(calls)
        assert nout.value == 0
        with pytest.raises(EngineError, match="EINVAL"):
            c16.feed(e, x[1000:1001])
        with pytest.raises(EngineError, match="EINVAL"):
            c16.feed(e, x[1000:3000], streams=[1, 1])
        with ch.Channelizer([0, 1, 2, 3], input_cs16=True) as wide:  # more channels than the engine has streams
            with pytest.raises(EngineError, match="EINVAL"):
                wide.feed(e, x)
        assert c16.pushed == 500 and c8.pushed == 500
        torch.cuda.synchronize()
        # a valid feed then continues the stream where the first push left it
        c16.feed(e, x[1000:60000], streams=[2, 0])
        e.process()
        r16 = c16.push(x[60000:])
        r8 = c8.push(cu8[1000:])
    assert np.array_equal(f16, w16[:, : f16.shape[1]]) and np.array_equal(r16, w16[:, 2 * ch.stream_outputs(0, 60000):])
    assert np.array_equal(np.concatenate([f8, r8], axis=1), w8)
