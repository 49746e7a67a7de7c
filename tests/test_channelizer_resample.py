"""The wideband channeliser's rate stage (include/nrsc5_b200.h: nrsc5b_chan_create_rate*): a capture at the radio's own
rate through an exact polyphase resampler in front of the FM and AM plans.  CPU tier: L, M and the offset limit against
integer arithmetic, the refused rates, the phase table (exact unit gain per phase, int16 taps, the int32 bound), the
reassembled prototype's response, the compiler's register report for k_resample, and the numpy restatement
(tests/chan_oracle_resample.py) on known signals.  GPU tier: k_resample and whole handles against the restatement bit
for bit, cu8 against cs16, streamed against one-shot, fs == R against the plain plan, synthetic stations decoding at
10 MS/s, 2.4 MS/s and 912 kS/s, and the feed into engines."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest

import chan_oracle_resample as rso
from nrsc5_b200 import channelizer as ch
from nrsc5_b200.engine import EngineError

EINVAL = -2
FM, AM = 0, 1
RATES_FM = [2048000, 2400000, 2500000, 3000000, 6000000, 8000000, 10000000, 20000000, 30720000, 61440000]
RATES_AM = [768000, 912000, 2400000]
PLAN_LIMIT = {(FM, 8): 29, (FM, 16): 59, (FM, 32): 0, (AM, 32): 74}        # the plans' own offset limits (0: none)
# (rate, decim, band) of the handles the GPU tier runs
HANDLES = [(10000000, 16, "fm"), (20000000, 32, "fm"), (2400000, 8, "fm"), (6000000, 8, "fm"), (61440000, 32, "fm"),
           (912000, 32, "am")]


def _expected(mode, decim, fs):
    """(L, M, max_offset) by exact integer arithmetic, or None where the library must refuse the rate."""
    r2 = 2976750 if mode == AM else decim * 1488375
    f2 = 2 * fs
    if fs <= 0 or 64 * fs < r2 or f2 > 4 * r2:
        return None
    g = math.gcd(r2, f2)
    L, M = r2 // g, f2 // g
    if L > 11907:
        return None
    lim = PLAN_LIMIT[(mode, decim)]
    if L == 1 == M:
        return L, M, lim
    step, half = (10000, 15000) if mode == AM else (100000, 200000)
    fp512 = 128 * min(f2, r2) - 22 * fs
    if fp512 < 512 * half:
        return None
    mo = (fp512 - 512 * half) // (512 * step)
    return L, M, min(mo, lim) if lim else mo


def _cases():
    return [(FM, d, r) for d in (8, 16, 32) for r in RATES_FM] + [(AM, 32, r) for r in RATES_AM]


def _counts(mode, decim, fs):
    L_, M_, mo = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    rc = ch._lib().nrsc5b_chan_resampler_tables(mode, decim, fs, ctypes.byref(L_), ctypes.byref(M_), ctypes.byref(mo), None)
    return rc, (L_.value, M_.value, mo.value)


def _band(mode):
    return "am" if mode == AM else "fm"


def _plan_rate(band, decim):
    return 1488375.0 if band == "am" else decim * 744187.5


# ---------------------------------------------------------------- CPU tier

def test_counts_match_integer_arithmetic():
    taken = 0
    for mode, decim, fs in _cases():
        want = _expected(mode, decim, fs)
        rc, got = _counts(mode, decim, fs)
        if want is None:
            assert rc == EINVAL, (mode, decim, fs)
            assert ch._lib().nrsc5b_chan_outputs_rate(mode, decim, fs, 1 << 20) == EINVAL
        else:
            assert rc == 0 and got == want, (mode, decim, fs, got, want)
            taken += 1
    assert taken >= 28
    # the rates the radios in the field run at, each with room for channels
    for mode, decim, fs, at_least in ((FM, 16, 10000000, 43), (FM, 8, 2400000, 8), (FM, 8, 6000000, 25), (FM, 32, 20000000, 89),
                                      (FM, 32, 61440000, 90), (AM, 32, 912000, 40), (AM, 32, 768000, 33)):
        assert _counts(mode, decim, fs)[1][2] >= at_least
    # fs == R: the plan itself
    for mode, decim, fs in ((FM, 8, 5953500), (FM, 16, 11907000), (FM, 32, 23814000), (AM, 32, 1488375)):
        assert _counts(mode, decim, fs) == (0, (1, 1, PLAN_LIMIT[(mode, decim)]))
        for t in (0, 63, 256, 100000):
            assert ch._lib().nrsc5b_chan_outputs_rate(mode, decim, fs, t) == ch.stream_outputs(0, 2 * t, _band(mode), decim)


def test_refused_rates_and_offsets_without_a_device():
    L = ch._lib()
    vp = ctypes.c_void_p
    off = np.array([0], dtype=np.int32)
    refused = [(FM, 16, 10000001),            # L > 11 907
               (FM, 8, 23814001 + 1),          # fs > 4 R
               (FM, 16, 11907000 // 32 - 500), # fs < R / 32
               (FM, 32, 0), (AM, 32, 0),
               (AM, 32, 1488375 * 4 + 125),
               (FM, 24, 10000000), (AM, 16, 912000), (2, 32, 912000)]
    for mode, decim, fs in refused:
        assert _counts(mode, decim, fs)[0] == EINVAL, (mode, decim, fs)
        assert L.nrsc5b_chan_outputs_rate(mode, decim, fs, 1000) == EINVAL
        for create in (L.nrsc5b_chan_create_rate, L.nrsc5b_chan_create_rate_cs16):
            h = vp()
            assert create(ctypes.byref(h), 0, mode, decim, fs, off.ctypes.data, 1) == EINVAL and not h.value
    for mode, decim, fs in ((FM, 16, 10000000), (FM, 8, 2400000), (AM, 32, 912000)):
        mo = _counts(mode, decim, fs)[1][2]
        for bad in ([mo + 1], [-mo - 1], [0, 3, mo + 1]):
            b = np.array(bad, dtype=np.int32)
            for create in (L.nrsc5b_chan_create_rate, L.nrsc5b_chan_create_rate_cs16):
                h = vp()
                assert create(ctypes.byref(h), 0, mode, decim, fs, b.ctypes.data, b.size) == EINVAL and not h.value
        h = vp()
        assert L.nrsc5b_chan_create_rate(ctypes.byref(h), 0, mode, decim, fs, None, 1) == EINVAL
        assert L.nrsc5b_chan_create_rate(ctypes.byref(h), 0, mode, decim, fs, off.ctypes.data, 0) == EINVAL
    with pytest.raises(ValueError):
        ch.resampler_tables(10000001, decim=16)
    with pytest.raises(ValueError):
        ch.resampler_tables(2.5e6 + 0.5, decim=16)
    with pytest.raises(ValueError):
        ch.outputs(6400, decim=16, rate=0)


def _listed():
    return [(m, d, r) for m, d, r in _cases() if _expected(m, d, r) is not None and _expected(m, d, r)[0] > 1]


@pytest.mark.parametrize("mode,decim,fs", _listed())
def test_phase_table(mode, decim, fs):
    """Every phase sums to exactly 2^14, every tap is int16, sum |G| < 2^16 per phase (the kernel's int32 bound); the
    reassembled prototype is within 0.01 dB up to f_p and at least 80 dB down from min(fs, R) - f_p on."""
    band = _band(mode)
    L, M, mo, G = ch.resampler_tables(fs, decim, band)
    assert G.shape == (L, 64) and G.dtype == np.int16
    g = G.astype(np.int64)
    assert np.all(g.sum(axis=1) == 1 << 14)
    sabs = np.abs(g).sum(axis=1)
    assert sabs.max() < 1 << 16
    assert (1 << 15) * sabs.max() + (1 << 13) < 1 << 31
    h = np.zeros(64 * L)
    for j in range(64):
        h[np.arange(L) + (63 - j) * L] = g[:, j]
    nf = 1 << int(np.ceil(np.log2(4 * h.size)))
    H = np.abs(np.fft.rfft(h, nf)) / (L * 2 ** 14)
    f = np.arange(H.size) * (L * fs) / nf
    R = _plan_rate(band, decim)
    fp = (min(fs, R) - 11 * fs / 128) / 2
    assert np.abs(20 * np.log10(H[f <= fp])).max() < 0.01
    assert H[f >= min(fs, R) - fp].max() < 10 ** (-80 / 20)


def test_k_resample_has_no_spills_and_no_stack(tmp_path):
    """-Xptxas -v on the channeliser: k_resample in both formats keeps everything in registers."""
    from nrsc5_b200 import build as b
    src = os.path.join(b.CSRC, "channelizer.cu")
    r = subprocess.run([os.environ.get("NVCC", "nvcc"), *b.ARCH, *b.COMMON, "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "c.o")],
                       capture_output=True, text=True, check=True)
    lines = r.stderr.splitlines()
    seen = 0
    for i, line in enumerate(lines):
        if "Function properties for" in line and "k_resample" in line:
            assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in lines[i + 1], lines[i + 1]
            seen += 1
    assert seen == 2


def _tone(m, step, amp, n, fs, cs16=False, phase=0.3):
    z = amp * np.exp(1j * (2 * np.pi * m * step / fs * np.arange(n) + phase))
    a = np.empty(2 * n)
    a[0::2], a[1::2] = z.real, z.imag
    if cs16:
        return np.clip(np.rint(a), -32768, 32767).astype(np.int16)
    return np.clip(np.rint(a + 127), 0, 255).astype(np.uint8)


@pytest.mark.parametrize("fs,decim,band", [(10000000, 16, "fm"), (2400000, 8, "fm"), (912000, 32, "am")])
def test_restatement_moves_a_tone_to_dc_and_rejects_the_neighbour(fs, decim, band):
    L, M, mo, G = ch.resampler_tables(fs, decim, band)
    step = 10e3 if band == "am" else 100e3
    m = mo - 2
    offs = [m, m - 6]
    taps, ph = ch.make_tables(offs, band=band, decim=decim)
    nout = 1500
    n = int(((nout + 2) * decim + (512 if band == "am" else 256)) * M / L) + 200
    x = _tone(m, step, 4000.0, n, fs, cs16=True)
    y = rso.channelize(x, offs, G, L, M, taps, ph, band, decim).astype(np.float64)
    z0 = y[0, 0::2] + 1j * y[0, 1::2]
    z1 = y[1, 0::2] + 1j * y[1, 1::2]
    assert z0.size >= nout
    assert abs(np.abs(z0).mean() - 4000.0) < 0.01 * 4000                  # unit gain through both stages
    assert np.abs(z0 - z0.mean()).max() < 0.01 * 4000                     # a constant: the tone sits at DC
    assert np.sqrt(np.mean(np.abs(z1) ** 2)) < 4000.0 * 10 ** (-60 / 20)   # the channel 600 kHz (60 kHz) away rejects it


@pytest.mark.parametrize("fs,decim,band", [(10000000, 16, "fm"), (61440000, 32, "fm"), (768000, 32, "am")])
def test_restatement_constant_in_constant_out(fs, decim, band):
    L, M, _, G = ch.resampler_tables(fs, decim, band)
    for v in ((1234, -567), (32767, -32768), (-20000, 0)):
        x = np.tile(np.array(v, dtype=np.int16), 5000)
        y = rso.resample(x, G, L, M)
        assert y.size == 2 * rso.resampled_of(5000, L, M) > 0
        assert np.all(y[0::2] == v[0]) and np.all(y[1::2] == v[1])         # exact unit gain per phase
    cu8 = np.tile(np.array([200, 31], dtype=np.uint8), 3000)
    y = rso.resample(cu8, G, L, M)
    assert np.all(y[0::2] == 64 * (200 - 127)) and np.all(y[1::2] == 64 * (31 - 127))


@pytest.mark.parametrize("fs,decim,band", [(2400000, 8, "fm"), (912000, 32, "am")])
def test_restatement_cu8_is_cs16_on_scaled_input(fs, decim, band):
    rng = np.random.default_rng(3)
    L, M, mo, G = ch.resampler_tables(fs, decim, band)
    offs = [-mo, 0, mo]
    taps, ph = ch.make_tables(offs, band=band, decim=decim)
    cu8 = rng.integers(0, 256, 2 * 60000, dtype=np.uint8)
    cu8[:200], cu8[200:400] = 0, 255
    x16 = (64 * (cu8.astype(np.int16) - 127)).astype(np.int16)
    assert np.array_equal(rso.resample(cu8, G, L, M), rso.resample(x16, G, L, M))
    assert np.array_equal(rso.channelize(cu8, offs, G, L, M, taps, ph, band, decim), rso.channelize(x16, offs, G, L, M, taps, ph, band, decim))


def _splits(nvalues, rng, big=(20000, 200000)):
    """Cut points into pushes of every awkward kind: empty, one sample, shorter than a window, odd sample counts, large."""
    cuts, pos, i = [0], 0, 0
    while pos < nvalues:
        step = [0, 2, 2 * int(rng.integers(1, 64)), 2 * int(rng.integers(64, 3000)) + 2, 2 * int(rng.integers(*big))][i % 5]
        pos = min(nvalues, pos + step)
        cuts.append(pos)
        i += 1
    return list(zip(cuts[:-1], cuts[1:]))


@pytest.mark.parametrize("fs,decim,band", [(10000000, 16, "fm"), (2400000, 8, "fm"), (912000, 32, "am")])
def test_restated_stream_equals_one_shot(fs, decim, band):
    rng = np.random.default_rng(11)
    L, M, mo, G = ch.resampler_tables(fs, decim, band)
    offs = [-mo, 1, mo]
    taps, ph = ch.make_tables(offs, band=band, decim=decim)
    nvalues = 2 * int(rng.integers(150000, 200000))
    x = rng.integers(-32768, 32768, nvalues, dtype=np.int16)
    parts = _splits(nvalues, rng)
    ys = rso.resample_stream([x[a:b] for a, b in parts], G, L, M)
    assert np.array_equal(np.concatenate(ys), rso.resample(x, G, L, M))
    outs = rso.channelize_stream([x[a:b] for a, b in parts], offs, G, L, M, taps, ph, band, decim)
    assert [o.shape[1] for o in outs] == [2 * ch.stream_outputs(a // 2, b - a, band, decim, fs) for a, b in parts]
    assert np.array_equal(np.concatenate(outs, axis=1), rso.channelize(x, offs, G, L, M, taps, ph, band, decim))


def test_channelizer_needs_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    for cs16 in (False, True):
        with pytest.raises(EngineError):
            ch.Channelizer([0, 9], input_cs16=cs16, decim=16, rate=10000000)
        with pytest.raises(EngineError):
            ch.Channelizer([0, 9], input_cs16=cs16, band="am", rate=912000)


# ---------------------------------------------------------------- GPU tier

def _full_range(rng, nvalues):
    x = rng.integers(-32768, 32768, nvalues, dtype=np.int16)
    x[rng.integers(0, nvalues, 64)] = -32768
    x[rng.integers(0, nvalues, 64)] = 32767
    return x


def _input(rng, nsamples, cs16):
    return _full_range(rng, 2 * nsamples) if cs16 else rng.integers(0, 256, 2 * nsamples, dtype=np.uint8)


def _first_diff(got, want):
    bad = np.argwhere(got != want)
    return f"{bad.shape[0]} of {got.size} values differ; first at {bad[:5].tolist()}: got {got[tuple(bad[0])]} want {want[tuple(bad[0])]}" \
        if bad.size else ""


@pytest.mark.gpu
@pytest.mark.parametrize("cs16", [False, True])
@pytest.mark.parametrize("fs,decim,band", [(10000000, 16, "fm"), (2400000, 8, "fm"), (61440000, 32, "fm"), (912000, 32, "am")])
def test_resample_kernel_equals_the_restatement(fs, decim, band, cs16):
    """One output (T = 64), a partial tile, and a run past the phase wrap at L with a tail of a partial tile; cs16 over
    the whole range, so that y saturates."""
    rng = np.random.default_rng(fs % 1000 + cs16)
    L, M, _, G = ch.resampler_tables(fs, decim, band)
    for T in (64, 64 + (300 * M) // L, (3 * L * M) // L + 4321):
        x = _input(rng, T, cs16)
        got = ch.resample(x, fs, decim, band)
        want = rso.resample(x, G, L, M)
        assert got.size == want.size == 2 * rso.resampled_of(T, L, M)
        assert not _first_diff(got, want), f"T = {T}: " + _first_diff(got, want)
        if cs16 and T > 1000:                                             # full-scale input: y saturates
            assert np.abs(want.astype(np.int32)).max() >= 32767


def _offsets(mo, nch, rng):
    if nch == "all" or nch >= 2 * mo + 1:
        return list(range(-mo, mo + 1))
    if nch == 1:
        return [int(rng.integers(-mo, mo + 1))]
    return [-mo] + [int(v) for v in rng.choice(np.arange(-mo + 1, mo), nch - 2, replace=False)] + [mo]


@pytest.mark.gpu
@pytest.mark.parametrize("nch", [1, 33, "all"])
@pytest.mark.parametrize("cs16", [False, True])
@pytest.mark.parametrize("fs,decim,band", HANDLES)
def test_handle_equals_the_restatement_bit_for_bit(fs, decim, band, cs16, nch):
    rng = np.random.default_rng(fs % 997 + 2 * cs16 + (nch if nch != "all" else 5))
    L, M, mo, G = ch.resampler_tables(fs, decim, band)
    offs = _offsets(mo, nch, rng)
    ntaps = 512 if band == "am" else 256
    nout = 64 * 9 + 13
    T = (((nout - 1) * decim + ntaps) * M) // L + 64 + 3
    x = _input(rng, T, cs16)
    with ch.Channelizer(offs, input_cs16=cs16, band=band, decim=decim, rate=fs) as c:
        taps, ph = c.tables()
        got = c.run(x)
    want = rso.channelize(x, offs, G, L, M, taps, ph, band, decim)
    assert got.shape == want.shape and got.shape[1] >= 2 * nout
    assert not _first_diff(got, want), _first_diff(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("fs,decim,band", [(10000000, 16, "fm"), (912000, 32, "am")])
def test_cu8_equals_cs16_on_scaled_input(fs, decim, band):
    rng = np.random.default_rng(21)
    mo = ch.resampler_tables(fs, decim, band)[2]
    offs = _offsets(mo, 9, rng)
    cu8 = rng.integers(0, 256, 2 * 400001, dtype=np.uint8)
    x16 = (64 * (cu8.astype(np.int16) - 127)).astype(np.int16)
    parts = _splits(x16.size, rng)
    with ch.Channelizer(offs, band=band, decim=decim, rate=fs) as c8, \
            ch.Channelizer(offs, input_cs16=True, band=band, decim=decim, rate=fs) as c16:
        want = c8.run(cu8)
        assert np.array_equal(c16.run(x16), want)
        s8 = np.concatenate([c8.push(cu8[a:b]) for a, b in parts], axis=1)
        s16 = np.concatenate([c16.push(x16[a:b]) for a, b in parts], axis=1)
    assert np.array_equal(s8, want) and np.array_equal(s16, want)
    assert np.array_equal(ch.resample(cu8, fs, decim, band), ch.resample(x16, fs, decim, band))


@pytest.mark.gpu
@pytest.mark.parametrize("cs16", [False, True])
@pytest.mark.parametrize("fs,decim,band", [(2400000, 8, "fm"), (61440000, 32, "fm"), (912000, 32, "am")])
def test_streamed_equals_one_shot_from_every_kind_of_memory(fs, decim, band, cs16):
    """Awkward splits from pageable, page-locked and device memory, the plan's mixer and the stage's phase wrapping
    inside the stream; then reset and the same again."""
    import torch
    rng = np.random.default_rng(200 + cs16 + fs % 1000)
    mo = ch.resampler_tables(fs, decim, band)[2]
    offs = _offsets(mo, 5, rng)
    nvalues = 2 * 700001
    x = _input(rng, nvalues // 2, cs16)
    item = 2 if cs16 else 1
    parts = _splits(nvalues, rng)
    nout = ch.stream_outputs(0, nvalues, band, decim, fs)
    d_x = torch.from_numpy(x).cuda()
    h_x = torch.from_numpy(x).pin_memory()
    with ch.Channelizer(offs, input_cs16=cs16, band=band, decim=decim, rate=fs) as c:
        whole = c.run(x)
        assert whole.shape[1] == 2 * nout
        d_one = torch.zeros((len(offs), 2 * nout + 64), dtype=torch.int16, device="cuda")
        c.run_device(d_x.data_ptr(), nvalues, d_one.data_ptr(), d_one.shape[1])
        torch.cuda.synchronize()
        assert np.array_equal(d_one[:, : 2 * nout].cpu().numpy(), whole)
        for rep in range(2):
            if rep:
                c.reset()
                assert c.pushed == 0
            d_out = torch.zeros((len(offs), 2 * nout + 64), dtype=torch.int16, device="cuda")
            col = 0
            for i, (a, b) in enumerate(parts):
                if i % 3 == 0:
                    got = c.push(x[a:b])
                    d_out[:, col: col + got.shape[1]] = torch.from_numpy(got).cuda()
                    col += got.shape[1]
                else:
                    src = d_x if i % 3 == 1 else h_x
                    n = c.push_device(src.data_ptr() + item * a, b - a, d_out.data_ptr() + 2 * col, d_out.shape[1])
                    col += 2 * n
            torch.cuda.synchronize()
            assert col == 2 * nout
            streamed = d_out[:, : 2 * nout].cpu().numpy()
            assert not _first_diff(streamed, whole), f"pass {rep}: " + _first_diff(streamed, whole)


@pytest.mark.gpu
@pytest.mark.parametrize("cs16", [False, True])
@pytest.mark.parametrize("fs,decim,band", [(2400000, 8, "fm"), (20000000, 32, "fm"), (912000, 32, "am")])
def test_one_shot_between_pushes_leaves_the_stream_alone(fs, decim, band, cs16):
    """push / one-shot on another capture (host and device entry) / push: the one-shot calls share the handle's planes
    with the stream, and the stream's outputs must still be the uninterrupted stream's, bit for bit."""
    import torch
    rng = np.random.default_rng(300 + cs16 + fs % 1000)
    mo = ch.resampler_tables(fs, decim, band)[2]
    offs = _offsets(mo, 5, rng)
    nvalues = 2 * 300001
    x = _input(rng, nvalues // 2, cs16)
    other = _input(rng, 150003, cs16)
    d_other = torch.from_numpy(other).cuda()
    nout_other = ch.outputs(other.size, band, decim, rate=fs)
    cuts = [0, 2 * 70001, 2 * 70001 + 2 * 33, 2 * 201117, nvalues]
    with ch.Channelizer(offs, input_cs16=cs16, band=band, decim=decim, rate=fs) as c:
        whole = c.run(x)
        parts = []
        for i, (a, b) in enumerate(zip(cuts[:-1], cuts[1:])):
            parts.append(c.push(x[a:b]))
            if i == 1:
                k = ch.resampled(b // 2, fs, decim, band)                 # a resampled carry is held here
                assert k - decim * ch.stream_outputs(0, b, band, decim, fs) > 0
                one = c.run(other)
                d_out = torch.zeros((len(offs), 2 * nout_other), dtype=torch.int16, device="cuda")
                c.run_device(d_other.data_ptr(), other.size, d_out.data_ptr(), 2 * nout_other)
                torch.cuda.synchronize()
                assert np.array_equal(d_out.cpu().numpy(), one)
            elif i == 2:
                c.resample_device(d_other.data_ptr(), other.size)
    streamed = np.concatenate(parts, axis=1)
    assert not _first_diff(streamed, whole), _first_diff(streamed, whole)


@pytest.mark.gpu
@pytest.mark.parametrize("cs16", [False, True])
def test_capture_larger_than_the_scratch(cs16):
    """2.4 MS/s -> D = 8 interpolates by 2.48: 3.5 M input samples are 8.7 M resampled ones, more than the planes hold, so
    one-shot and streamed both go through them in pieces; both equal the restatement at the start, across the first
    piece boundary and at the end."""
    import torch
    fs, decim = 2400000, 8
    rng = np.random.default_rng(31)
    L, M, mo, G = ch.resampler_tables(fs, decim)
    offs = [0, mo, -mo, 3]
    nvalues = 2 * 3500000
    x = _input(rng, nvalues // 2, cs16)
    nout = ch.outputs(nvalues, decim=decim, rate=fs)
    stride = 2 * nout + 32
    d_x = torch.from_numpy(x).cuda()
    with ch.Channelizer(offs, input_cs16=cs16, decim=decim, rate=fs) as c:
        taps, ph = c.tables()
        d_out = torch.zeros((len(offs), stride), dtype=torch.int16, device="cuda")
        c.run_device(d_x.data_ptr(), nvalues, d_out.data_ptr(), stride)
        torch.cuda.synchronize()
        one = d_out[:, : 2 * nout].cpu().numpy()
        got = np.concatenate([c.push(x[:302]), c.push(x[302: nvalues - 1000]), c.push(x[nvalues - 1000:])], axis=1)
    assert np.array_equal(got, one)
    y = ch.resample(x, fs, decim)
    assert y.size > 2 * ((1 << 22) + 256)
    for n0, n in ((0, 600), ((1 << 19) - 300, 600), (nout - 300, 300)):
        seg = y[2 * decim * n0: 2 * (decim * (n0 + n - 1) + 256)]
        want = rso.chan_oracle_rates.channelize(seg, offs, taps, ph, decim, n0=n0)
        assert np.array_equal(one[:, 2 * n0: 2 * (n0 + n)], want), f"outputs {n0} .. {n0 + n - 1}"
    assert np.array_equal(y[: 2 * 5000], rso.resample(x[: 2 * 3000], G, L, M)[: 2 * 5000])


@pytest.mark.gpu
@pytest.mark.parametrize("cs16", [False, True])
@pytest.mark.parametrize("fs,decim,band", [(11907000, 16, "fm"), (1488375, 32, "am")])
def test_rate_equal_to_the_plan_is_the_plan(fs, decim, band, cs16):
    rng = np.random.default_rng(5)
    offs = [-20, 0, 7, 20]
    x = _input(rng, 64 * 600, cs16)
    c = ch.Channelizer(offs, input_cs16=cs16, band=band, decim=decim, rate=fs)
    assert c.rate is None
    with c, ch.Channelizer(offs, input_cs16=cs16, band=band, decim=decim) as plain:
        assert np.array_equal(c.run(x), plain.run(x))
        assert np.array_equal(c.push(x[:3000]), plain.push(x[:3000]))


# ---- synthetic stations at the radio's rate, one-shot into an engine and fed straight into it

def _to_rate(z, rate_in, fs):
    """Band-limited resampling of a complex GPU tensor from rate_in to fs by FFT zero-padding or truncation: n is cut to a
    multiple of rate_in / gcd(rate_in, fs), so that the ratio is exact.  Independent of the library's filter."""
    import torch
    from fractions import Fraction
    ratio = Fraction(fs) / rate_in
    num, den = ratio.numerator, ratio.denominator
    n = (z.numel() // den) * den
    N = n // den * num
    X = torch.fft.fft(z[:n])
    Y = torch.zeros(N, dtype=torch.complex64, device=z.device)
    k = min(n, N) // 2
    Y[:k] = X[:k]
    Y[-k:] = X[-k:]
    return torch.fft.ifft(Y) * (N / n)


def _station_band(stations, fs, cs16, noise, step):
    """Each station's capture (cu8 or cs16 at rate_in, as a complex tensor) resampled to fs, moved to m x step and
    scaled; summed with noise and quantised.  Returns the capture as numpy (cs16 or cu8)."""
    import torch
    ys = [(_to_rate(z, r, fs), m, s) for z, r, m, s in stations]
    N = min(y.numel() for y, _, _ in ys)
    t = torch.arange(N, dtype=torch.float64, device="cuda")
    wide = torch.zeros(N, dtype=torch.complex64, device="cuda")
    for y, m, s in ys:
        phase = torch.remainder(t * (m * step / fs), 1.0) * (2 * math.pi)
        wide += y[:N] * s * torch.complex(torch.cos(phase).float(), torch.sin(phase).float())
    g = torch.Generator(device="cuda")
    g.manual_seed(fs % 1000)
    iq = torch.stack([wide.real, wide.imag], -1) + torch.randn((N, 2), generator=g, device="cuda") * noise
    if cs16:
        x = torch.clamp(torch.round(iq), -32768, 32767).to(torch.int16)
    else:
        x = torch.clamp(torch.round(iq + 127), 0, 255).to(torch.uint8)
    return x.reshape(-1).cpu().numpy()


def _fm_z(cap):
    import torch
    xi = torch.from_numpy(cap.cu8.astype(np.float32) - 127.0).cuda().view(-1, 2)
    return torch.complex(xi[:, 0].contiguous(), xi[:, 1].contiguous())


def _fm_band(fs, cs16):
    from fractions import Fraction
    from nrsc5_b200 import synth
    if cs16:                                                              # three MP1 stations 48 dB apart
        spec = [(11, 250.0, 90, 40), (-23, 1.0, 91, 540), (-21, 60.0, 93, 1540)]
        noise = 2.0
    else:                                                                 # two that 8 bits hold without clipping
        spec = [(4, 0.6, 70, 540), (-5, 0.6, 71, 940)]
        noise = 2.0
    caps = [synth.make_fm_mp1(nframes=1, seed=seed, lead_in=lead, tail_blocks=3) for _, _, seed, lead in spec]
    st = [(_fm_z(c), Fraction(1488375), m, s) for c, (m, s, _, _) in zip(caps, spec)]
    return [m for m, _, _, _ in spec], _station_band(st, fs, cs16, noise, 100e3), caps


def _am_band(fs):
    import torch
    from fractions import Fraction
    from nrsc5_b200 import synth_am
    spec = [(-17, 0.3, False), (12, 1.0, True)]                           # one MA1, one MA3 10 dB above it
    caps = [synth_am.make_am_ma1(nframes=7, seed=400 + i, lead_in=300 + 200 * i, psmi=2 if ma3 else 1) for i, (_, _, ma3) in enumerate(spec)]
    st = []
    for c, (m, s, _) in zip(caps, spec):
        xi = torch.from_numpy(c.cs16.astype(np.float32)).cuda().view(-1, 2)
        st.append((torch.complex(xi[:, 0].contiguous(), xi[:, 1].contiguous()), Fraction(1488375, 32), m, s))
    return [m for m, _, _ in spec], _station_band(st, fs, True, 3.0, 10e3), caps, spec


def _one_shot_records(x, offs, fs, decim, band, cs16):
    """nrsc5b_chan_run_device* on the whole capture, the engine attached to its output, one nrsc5b_process."""
    import torch
    import nrsc5_b200
    d_x = torch.from_numpy(x).cuda()
    nout = ch.outputs(x.size, band, decim, rate=fs)
    stride = (2 * nout + 64) & ~31
    d_out = torch.zeros((len(offs), stride), dtype=torch.int16, device="cuda")
    with ch.Channelizer(offs, input_cs16=cs16, band=band, decim=decim, rate=fs) as c:
        c.run_device(d_x.data_ptr(), x.size, d_out.data_ptr(), stride)
        torch.cuda.synchronize()
    kw = dict(mode="am") if band == "am" else {}
    with nrsc5_b200.Engine(nstreams=len(offs), input_capacity=4096, log_capacity=8 << 20, input_cs16=True, **kw) as e:
        if band == "am":
            e.enable_l2()
        e.attach_device_input(d_out.data_ptr(), 2 * stride, 4 * nout)
        e.process()
        recs = [_drain(e, band, s) for s in range(len(offs))]
    return d_out[:, : 2 * nout].cpu().numpy(), recs


def _check_fm(x, offs, fs, decim, caps, y, recs):
    import port
    from nrsc5_b200 import engine as eng, synth
    L, M, _, G = ch.resampler_tables(fs, decim)
    taps, ph = ch.make_tables(offs, decim=decim)
    head = rso.channelize(x[: 2 * ((3000 * decim + 256) * M // L + 70)], offs, G, L, M, taps, ph, "fm", decim)
    assert np.array_equal(y[:, : 2 * 3000], head[:, : 2 * 3000])
    for s in range(len(offs)):
        p1 = [r["bits"] for t_, r in recs[s] if t_ == eng.REC_FRAME and r["lc"] == 0]
        assert any(synth.pack_bits(f) in p1 for f in caps[s].p1_frames), f"station {s}: its P1 PDU did not come out"
        ref = port.decode(y[s])
        assert p1 == ref.p1_frames, f"station {s}: P1 PDUs differ from the oracle's decode"
        assert [r["bits"] for t_, r in recs[s] if t_ == eng.REC_PIDS] == ref.pids_frames


@pytest.mark.gpu
def test_fm_stations_at_10_msps_cs16_decode():
    offs, x, caps = _fm_band(10000000, True)
    assert np.abs(x).max() > 20000
    y, recs = _one_shot_records(x, offs, 10000000, 16, "fm", True)
    _check_fm(x, offs, 10000000, 16, caps, y, recs)


@pytest.mark.gpu
def test_fm_stations_at_2_4_msps_cu8_decode():
    offs, x, caps = _fm_band(2400000, False)
    assert x.dtype == np.uint8
    y, recs = _one_shot_records(x, offs, 2400000, 8, "fm", False)
    _check_fm(x, offs, 2400000, 8, caps, y, recs)


@pytest.mark.gpu
def test_am_stations_at_912_ksps_decode():
    import test_channelizer_am as tam
    offs, x, caps, spec = _am_band(912000)
    y, raw = _one_shot_records(x, offs, 912000, 32, "am", True)
    L, M, _, G = ch.resampler_tables(912000, band="am")
    taps, ph = ch.make_tables(offs, band="am")
    head = rso.channelize(x[: 2 * ((2000 * 32 + 512) * M // L + 70)], offs, G, L, M, taps, ph, "am")
    assert np.array_equal(y[:, : 2 * 2000], head[:, : 2 * 2000])
    for s, (_, _, ma3) in enumerate(spec):
        tam._check_station(raw[s], y[s], caps[s], ma3)


def _without_positions(recs):
    from nrsc5_b200 import engine as eng
    return [(t, {k: v for k, v in r.items() if not (t == eng.REC_BLOCK and k == "start")}) for t, r in recs]


def _ragged(nvalues, seed):
    rng = np.random.default_rng(seed)
    cuts, pos = [0], 0
    while pos < nvalues:
        pos = min(nvalues, pos + (2 * int(rng.integers(1, 300)) if rng.random() < 0.2 else 2 * int(rng.integers(1 << 18, 3 << 19))))
        cuts.append(pos)
    return list(zip(cuts[:-1], cuts[1:]))


@pytest.fixture(scope="module", params=["fm", "am"])
def fed_band(request):
    if request.param == "fm":
        offs, x, _ = _fm_band(10000000, True)
        fs, decim = 10000000, 16
    else:
        offs, x, _, _ = _am_band(912000)
        fs, decim = 912000, 32
    _, ref = _one_shot_records(x, offs, fs, decim, request.param, True)
    return request.param, offs, x, fs, decim, ref


def _engine(band, n, cap):
    import nrsc5_b200
    kw = dict(mode="am") if band == "am" else {}
    e = nrsc5_b200.Engine(nstreams=n, input_capacity=cap, log_capacity=8 << 20, input_cs16=True, **kw)
    if band == "am":
        e.enable_l2()
    return e


def _drain(e, band, s):
    """The stream's new records; AM (with L2 on the device): every REC_L2 moved behind its frame, so that the order does
    not depend on how the input was cut into nrsc5b_process calls."""
    from nrsc5_b200 import engine as eng
    return eng.with_l2_in_call_order(e.drain_raw(s)) if band == "am" else e.drain(s)


@pytest.mark.gpu
def test_feed_with_permuted_streams_and_trims(fed_band):
    band, offs, x, fs, decim, ref = fed_band
    n = len(offs)
    nout = ch.outputs(x.size, band, decim, rate=fs)
    perm = list(range(n))[::-1]
    with ch.Channelizer(offs, input_cs16=True, band=band, decim=decim, rate=fs) as c, _engine(band, n, 4 * nout + 4096) as e:
        got = [[] for _ in offs]
        for a, b in _ragged(x.size, 1):
            c.feed(e, x[a:b], streams=perm)                               # channel k -> stream perm[k]
            e.process()
            for k in range(n):
                got[k] += _drain(e, band, perm[k])
    assert got == ref
    cap = 1 << 20 if band == "am" else 3 << 20
    assert 4 * nout > cap
    recs = [[] for _ in offs]
    with ch.Channelizer(offs, input_cs16=True, band=band, decim=decim, rate=fs) as c, _engine(band, n, cap) as e:
        for a, b in _ragged(x.size, 2):
            c.feed(e, x[a:b])
            e.process()
            for s in range(n):
                recs[s] += _drain(e, band, s)
    assert [_without_positions(r) for r in recs] == [_without_positions(r) for r in ref]


@pytest.mark.gpu
def test_feed_back_pressure_is_all_or_nothing(fed_band):
    import torch
    band, offs, x, fs, decim, ref = fed_band
    n = len(offs)
    host = torch.from_numpy(x).pin_memory()
    L, M, _, _ = ch.resampler_tables(fs, decim, band)
    step = 2 * ((1 << 19) * decim // 32 * M // L)                        # int16 values per push: about 2^19 / 32 x D resampled samples
    refused = 0
    recs = [[] for _ in offs]
    with ch.Channelizer(offs, input_cs16=True, band=band, decim=decim, rate=fs) as c, _engine(band, n, 1 << 20) as e:
        pos, processing = 0, False
        while pos < x.size:
            k = min(step, x.size - pos)
            before = c.pushed
            try:
                c.feed(e, (host.data_ptr() + 2 * pos, k))
            except EngineError as ex:
                assert "EFULL" in str(ex) and not processing
                assert c.pushed == before
                refused += 1
                processing = True
                e.process()
                for s in range(n):
                    recs[s] += _drain(e, band, s)
                c.feed(e, (host.data_ptr() + 2 * pos, k))
            pos += k
            if processing:
                e.process()
                for s in range(n):
                    recs[s] += _drain(e, band, s)
        e.process()
        for s in range(n):
            recs[s] += _drain(e, band, s)
        torch.cuda.synchronize()
    assert refused == 1
    assert [_without_positions(r) for r in recs] == [_without_positions(r) for r in ref]


@pytest.mark.gpu
def test_one_shot_between_feeds_leaves_the_stream_alone(fed_band):
    """feed / one-shot on another capture / feed: the records equal the one-shot path's, stream for stream."""
    band, offs, x, fs, decim, ref = fed_band
    n = len(offs)
    nout = ch.outputs(x.size, band, decim, rate=fs)
    rng = np.random.default_rng(8)
    other = _full_range(rng, 2 * 200001)
    recs = [[] for _ in offs]
    with ch.Channelizer(offs, input_cs16=True, band=band, decim=decim, rate=fs) as c, _engine(band, n, 4 * nout + 4096) as e:
        for i, (a, b) in enumerate(_ragged(x.size, 3)):
            c.feed(e, x[a:b])
            e.process()
            for s in range(n):
                recs[s] += _drain(e, band, s)
            if i % 2 == 0:
                assert c.run(other).shape[1] > 0
    assert recs == ref
