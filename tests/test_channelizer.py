"""Wideband channeliser (SURVEY 8 f3; csrc/channelizer.cu).  CPU tier: the definition's tables (filter quality) and its
numpy restatement on signals with known answers.  GPU tier: the wgmma kernel against the restatement, bit for bit,
and end to end - stations mixed into a 23.814 MS/s capture come out of channeliser + engine with their PDUs intact."""
import numpy as np
import pytest

import chan_oracle
from nrsc5_b200 import channelizer as ch

WIDE = ch.WIDE_RATE


def test_tables_filter_quality_and_symmetry():
    taps, ph = ch.make_tables([0, 9, -37])
    assert np.abs(ph.astype(np.int64)[:, 0] ** 2 + ph.astype(np.int64)[:, 1] ** 2 - 32767 ** 2).max() < 2 * 32767 * 2
    assert np.array_equal(ph[1:, 0], ph[:0:-1, 0]) and np.array_equal(ph[1:, 1], -ph[:0:-1, 1])   # P[N - i] = conj(P[i])
    h = taps[0, :, 0].astype(np.float64)                                  # channel 0: no mixing, real taps
    assert np.all(taps[0, :, 1] == 0) and abs(h.sum() - 2 ** 19) < 64     # unit DC gain at the 2^19 scale
    H = np.abs(np.fft.fft(h, 1 << 16)) / h.sum()
    f = np.fft.fftfreq(1 << 16, 1 / WIDE)
    assert H[np.abs(f) <= 200e3].min() > 0.97                             # flat over a hybrid FM channel (+-200 kHz)
    assert H[np.abs(f) >= 544e3].max() < 10 ** (-55 / 20)                 # what would alias onto it after /32: >= 55 dB down
    # a mixed channel's taps are the prototype times the table's phasor: same magnitudes within rounding
    mag = np.hypot(taps[1, :, 0].astype(float), taps[1, :, 1].astype(float))
    assert np.abs(mag - np.abs(h[::1])).max() <= 1.5
    assert np.abs(taps.astype(np.int64)).max() <= 127 * 256 + 127          # both bytes of every tap are int8 (the tensor-core operand)


def _tone(m_100khz, amp, n, phase=0.3):
    t = np.arange(n)
    x = amp * np.exp(1j * (2 * np.pi * m_100khz * 100e3 / WIDE * t + phase))
    a = np.empty(2 * n, dtype=np.uint8)
    a[0::2] = np.clip(np.rint(x.real + 127), 0, 255)
    a[1::2] = np.clip(np.rint(x.imag + 127), 0, 255)
    return a


def test_oracle_moves_a_tone_at_the_channel_centre_to_dc():
    offs = [17, -5]
    taps, ph = ch.make_tables(offs)
    cu8 = _tone(17, 50.0, 32 * 600)
    y = chan_oracle.channelize(cu8, offs, taps, ph).astype(np.float64)
    z0 = y[0, 0::2] + 1j * y[0, 1::2]
    z1 = y[1, 0::2] + 1j * y[1, 1::2]
    assert abs(np.abs(z0).mean() - 50.0 * 64) < 0.02 * 50 * 64            # unit gain: 64 LSB per input LSB
    assert np.abs(z0 - z0.mean()).max() < 0.02 * 50 * 64                  # a constant: the tone sits at DC of channel 17
    assert np.abs(z1).max() < 50.0 * 64 * 10 ** (-48 / 20)                # and is rejected by the channel 2.2 MHz away (what is left is the
                                                                          # rounding noise of the 8-bit input that falls into that channel)


@pytest.mark.gpu
@pytest.mark.parametrize("nch,nbytes", [(3, 64 * 700), (40, 64 * 1031), (33, 64 * 135), (5, 64 * 25001)])   # the last: the mixer wraps twice
def test_kernel_equals_the_restatement_bit_for_bit(nch, nbytes):
    rng = np.random.default_rng(nch)
    offs = list(rng.choice(np.arange(-118, 119), nch, replace=False))
    cu8 = rng.integers(0, 256, nbytes, dtype=np.uint8)
    with ch.Channelizer(offs) as c:
        taps, ph = c.tables()
        t2, p2 = ch.make_tables(offs)
        assert np.array_equal(taps, t2) and np.array_equal(ph, p2)
        got = c.run(cu8)
    want = chan_oracle.channelize(cu8, offs, taps, ph)
    assert got.shape == want.shape
    bad = np.argwhere(got != want)
    assert bad.size == 0, f"{bad.shape[0]} of {got.size} values differ; first at (channel, value) {bad[:5].tolist()}: " \
                          f"got {got[tuple(bad[0])]} want {want[tuple(bad[0])]}"


@pytest.mark.gpu
def test_stations_in_a_wideband_capture_decode_bit_exact():
    """Two synthetic FM MP1 stations 1.1 MHz and -2.3 MHz from the capture centre (plus noise), 23.814 MS/s cu8 ->
    channeliser -> two cs16 streams -> engine: the PDUs are the ones the generator put in, and equal to what the CPU
    oracle decodes from the restatement's output of the same capture."""
    import scipy.fft
    import port
    import nrsc5_b200
    from nrsc5_b200 import engine as eng, synth
    offs = [11, -23]
    caps = [synth.make_fm_mp1(nframes=1, seed=70 + i, lead_in=900 * i + 40, tail_blocks=3) for i in range(2)]
    n = min(c.cu8.size for c in caps) // 2
    up = 16
    wide = np.zeros(n * up, dtype=np.complex64)
    t = np.arange(n * up, dtype=np.float64)
    for c, m in zip(caps, offs):
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
    cu8 = cu8[: cu8.size & ~63]
    with ch.Channelizer(offs) as c:
        taps, ph = c.tables()
        cs16 = c.run(cu8)
    # a slice of the device output against the restatement (the whole capture is 80 M samples: one block's worth here)
    part = cu8[: 64 * 4000]
    want = chan_oracle.channelize(part, offs, taps, ph)
    assert np.array_equal(cs16[:, : want.shape[1]], want)
    with nrsc5_b200.Engine(nstreams=2, input_capacity=2 * cs16.shape[1] + 4096, log_capacity=4 << 20, input_cs16=True) as e:
        for s in range(2):
            e.push_cs16(s, cs16[s])
        e.process()
        recs = [e.drain(s) for s in range(2)]
    for s in range(2):
        p1 = [r["bits"] for t_, r in recs[s] if t_ == eng.REC_FRAME and r["lc"] == 0]
        assert any(synth.pack_bits(f) in p1 for f in caps[s].p1_frames), f"station {s}: its P1 PDU did not come out"
        ref = port.decode(cs16[s])
        assert p1 == ref.p1_frames
        assert [r["bits"] for t_, r in recs[s] if t_ == eng.REC_PIDS] == ref.pids_frames
    # the same without leaving the GPU: the channeliser writes a device buffer that the engine reads in place
    import torch
    d_cu8 = torch.from_numpy(cu8).cuda()
    nout = ch.outputs(cu8.size)
    stride = (2 * nout + 64) & ~31                                       # int16 values between channels
    d_out = torch.zeros((2, stride), dtype=torch.int16, device="cuda")
    with ch.Channelizer(offs) as c:
        c.run_device(d_cu8.data_ptr(), cu8.size, d_out.data_ptr(), stride)
        torch.cuda.synchronize()
    with nrsc5_b200.Engine(nstreams=2, input_capacity=4096, log_capacity=4 << 20, input_cs16=True) as e:
        e.attach_device_input(d_out.data_ptr(), 2 * stride, 4 * nout)
        e.process()
        assert [e.drain(s) for s in range(2)] == recs
