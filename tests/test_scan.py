"""The band scan (include/nrsc5_b200.h: nrsc5b_scan_*, nrsc5b_chan_scan).  CPU tier: the published taps against their
stated response, c and kappa recomputed from their definitions, the numpy restatement (tests/scan_oracle.py) on
hand-built inputs, argument checks.  GPU tier: k_scan / k_scan_finish against the restatement bit for bit, streamed in
awkward pieces, FM and AM bands with stations, carriers, spurs and noise, nrsc5b_chan_scan against channelise-then-scan,
the sideband SNR against the truth, and no false alarm on noise."""
import math

import numpy as np
import pytest

import scan_oracle as so
from nrsc5_b200 import scan
from nrsc5_b200.engine import EngineError

FM, AM = 0, 1
C = {FM: 5.055, AM: 4.682}
C1 = {FM: 4.190, AM: 4.022}
KAPPA = {FM: 0.310, AM: 0.313}
BAND = {FM: "fm", AM: "am"}


def _iq(z):
    iq = np.empty(2 * z.size)
    iq[0::2] = z.real
    iq[1::2] = z.imag
    return np.clip(np.rint(iq), -32768, 32767).astype(np.int16)


def _fm_channel(seed=3, psmi=1, nframes=1, lead_in=0, cfo_hz=0.0, gain=64.0, tail_blocks=0):
    """A synthetic FM station (synth.make_fm, cu8 at 1 488 375 S/s) at the channel rate 744 187.5 S/s, complex, with
    `gain` cs16 LSB per cu8 LSB."""
    from scipy.signal import resample_poly
    from nrsc5_b200 import synth
    cap = synth.make_fm(psmi=psmi, nframes=nframes, seed=seed, lead_in=lead_in, cfo_hz=cfo_hz, tail_blocks=tail_blocks)
    x = cap.cu8.astype(np.float64) - 127.0
    return resample_poly(x[0::2] + 1j * x[1::2], 1, 2) * gain


# ---------------------------------------------------------------- CPU tier

def test_fm_taps_response():
    taps, kappa = scan.make_tables("fm")
    assert kappa == KAPPA[FM]
    fs, F = 744187.5, 2048
    f = np.linspace(-fs / 2, fs / 2, 40001)
    db = so.response_db(taps, f, fs)
    up = (f >= 356 * fs / F) & (f <= 478 * fs / F)
    assert db[up].max() - db[up].min() <= 0.5 and abs(db[up].mean()) < 0.25      # unit passband gain, flat
    assert db[np.abs(f) <= 100e3].max() <= -40.0                                 # the channel's analogue host
    assert db[f >= 202e3].max() <= -40.0                                         # a station 400 kHz away
    assert db[f <= -356 * fs / F].max() < -40.0                                  # the other sideband
    lo = np.stack([taps[:, 0], -taps[:, 1]], 1)                                  # g_L = conj(g_U): the mirror image
    assert np.allclose(so.response_db(lo, -f[up], fs), db[up])
    assert np.abs(taps[:, 0].astype(np.int64)).sum() < 1 << 16 and np.abs(taps[:, 1].astype(np.int64)).sum() < 1 << 16


def test_am_taps_response():
    taps, kappa = scan.make_tables("am")
    assert kappa == KAPPA[AM]
    fs = 46511.71875
    assert taps[:, 0].astype(np.int64).sum() == 0 and taps[:, 1].astype(np.int64).sum() == 0    # exact null at DC
    f = np.linspace(-fs / 2, fs / 2, 20001)
    db = so.response_db(taps, f, fs)
    flat = (f >= 6500) & (f <= 14000)
    assert db[flat].max() - db[flat].min() <= 0.5 and abs(db[flat].mean()) < 0.25
    assert db[np.abs(f) <= 5000].max() < -15.0 and db[np.abs(f) <= 3000].max() < -45.0
    assert np.abs(taps[:, 0].astype(np.int64)).sum() < 1 << 16 and np.abs(taps[:, 1].astype(np.int64)).sum() < 1 << 16


@pytest.mark.parametrize("mode", [FM, AM])
def test_c_is_its_derivation(mode):
    """c = sqrt(gamma ln(1e6 J) / 2), gamma from the published taps (the header's derivation)."""
    taps, _ = scan.make_tables(BAND[mode])
    _, _, q, _, J, _ = so.geometry(mode)
    assert abs(math.sqrt(so.gamma(taps, q) * math.log(1e6 * J) / 2) - C[mode]) < 1e-3


@pytest.mark.parametrize("mode", [FM, AM])
def test_c1_is_its_derivation(mode):
    """c1 = sqrt(gamma ln(1e3)): one sideband at one timing, noise alone passing once in a thousand."""
    taps, _ = scan.make_tables(BAND[mode])
    assert abs(math.sqrt(so.gamma(taps, so.geometry(mode)[2]) * math.log(1e3)) - C1[mode]) < 1e-3


def test_grid_offsets():
    assert scan.grid_offsets("fm") == list(range(-117, 118))
    assert scan.grid_offsets("fm", decim=16) == list(range(-59, 60))
    assert scan.grid_offsets("am") == list(range(-74, 75))
    assert scan.grid_offsets("fm", rate=23814000) == list(range(-117, 118))       # the plan's own rate
    assert scan.grid_offsets("fm", rate=10000000, decim=16) == list(range(-43, 44))


@pytest.mark.parametrize("mode", [FM, AM])
def test_one_sideband_of_a_station_beside_is_not_a_detection(mode):
    """A station's upper sideband alone, as it falls into the lower filter of the channel 300 kHz (AM: 20 kHz) above
    it, and the station itself: the combined score passes in both, but only the station holds both sidebands."""
    F, P, q, S, J, fs = so.geometry(mode)
    taps, kappa = scan.make_tables(BAND[mode])
    if mode == FM:
        y = _fm_channel(seed=5)[: int(0.6 * fs)]
        shift = 300e3
    else:
        from nrsc5_b200 import synth_am
        c = synth_am.make_am_ma3(nframes=2, seed=4, lead_in=0).cs16
        y = c[0::2] + 1j * c[1::2].astype(np.float64)
        shift = 20e3
    t = np.arange(y.size)
    Y = np.fft.fft(y)
    up = np.fft.ifft(Y * (np.fft.fftfreq(y.size) > 0))             # the station's upper half, then moved down
    rng = np.random.default_rng(2)
    # 30 dB under the station: far stronger ones leak through the filters' 40 dB stopbands into both sidebands
    noise = 0.03 * np.sqrt(np.mean(np.abs(y) ** 2) / 2) * (rng.standard_normal(y.size) + 1j * rng.standard_normal(y.size))
    _, res = so.scan(np.stack([_iq(y + noise), _iq(up * np.exp(-2j * np.pi * shift / fs * t) + noise)]), mode, taps, C[mode],
                     kappa, C1[mode])
    assert res[0]["detected"] and res[1]["score"] >= res[1]["threshold"]
    assert res[1]["score_lower"] >= res[1]["threshold_sideband"] and res[1]["score_upper"] < res[1]["score_lower"] / 4
    assert not res[1]["detected"]


def test_kappa_fm_from_a_noise_free_station():
    taps, kappa = scan.make_tables("fm")
    y = _iq(_fm_channel())
    _, res = so.scan(y[None], FM, taps, C[FM], kappa, C1[FM])
    assert abs((res[0]["rho_lower"] + res[0]["rho_upper"]) / 2 - kappa) < 1e-3
    assert res[0]["timing"] == 0 and res[0]["detected"]


def test_kappa_am_from_a_noise_free_station():
    from nrsc5_b200 import synth_am
    taps, kappa = scan.make_tables("am")
    y = synth_am.make_am_ma3(nframes=4, seed=3, lead_in=0).cs16
    _, res = so.scan(y[None], AM, taps, C[AM], kappa, C1[AM])
    assert abs((res[0]["rho_lower"] + res[0]["rho_upper"]) / 2 - kappa) < 1e-3
    assert res[0]["timing"] == 0 and res[0]["detected"]


@pytest.mark.parametrize("mode", [FM, AM])
def test_restatement_tone_and_noise_give_nothing(mode):
    F, P, q, S, J, fs = so.geometry(mode)
    taps, kappa = scan.make_tables(BAND[mode])
    n = 300 * S + F + 64                            # every fold position gets the same number of products
    t = np.arange(n)
    f_tone = (451 if mode == FM else 57) * fs / F + 37.0                  # inside the upper sideband
    tone = _iq(12000 * np.exp(2j * np.pi * f_tone / fs * t))
    rng = np.random.default_rng(5)
    noise = _iq(3000 * (rng.standard_normal(n) + 1j * rng.standard_normal(n)))
    acc, res = so.scan(np.stack([tone, noise]), mode, taps, C[mode], kappa, C1[mode])
    cw = so.windows(acc, mode)
    Cu = cw[0, 3] + 1j * cw[0, 4].astype(np.float64)
    assert np.abs(Cu - Cu.mean()).max() < 1e-5 * np.abs(Cu).max()       # the tone: constant over every timing
    assert res[0]["score"] < 1e-5
    assert res[1]["score"] < res[1]["threshold"] and not res[1]["detected"]
    assert res[1]["symbols"] > 32


@pytest.mark.parametrize("mode", [FM, AM])
def test_restatement_cp_sequence_gives_timing_and_cfo(mode):
    """A sequence of random OFDM-like symbols with their cyclic prefix: timing lands on the generated symbol start,
    and an applied frequency offset comes out as the difference of the estimates with and without it."""
    F, P, q, S, J, fs = so.geometry(mode)
    taps, kappa = scan.make_tables(BAND[mode])
    rng = np.random.default_rng(11)
    nsym, lead = 120, 5 * S + 3 * q
    body = rng.standard_normal((nsym, F)) + 1j * rng.standard_normal((nsym, F))
    x = np.concatenate([np.zeros(lead), np.concatenate([body[:, F - P:], body], 1).reshape(-1) * 3000])
    t = np.arange(x.size)
    off = 0.2 * fs / F
    ys = np.stack([_iq(x), _iq(x * np.exp(2j * np.pi * off / fs * t))])
    _, res = so.scan(ys, mode, taps, C[mode], kappa, C1[mode])
    assert res[0]["timing"] == lead % S and res[1]["timing"] == lead % S
    assert res[0]["detected"] and res[1]["detected"]
    assert abs(res[1]["cfo_hz"] - res[0]["cfo_hz"] - off) < 0.01                # Hz
    assert abs(res[0]["cfo_hz"]) < 0.01 * fs / F                                 # the random symbols' own spread


def test_scan_needs_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(EngineError, match="ENODEV"):
        scan.Scanner(4)


def test_argument_checks_without_a_device():
    with pytest.raises(ValueError):
        scan.make_tables("dab")
    L = scan._lib()
    import ctypes
    assert L.nrsc5b_scan_make_tables(2, None, None) == -2
    h = ctypes.c_void_p()
    assert L.nrsc5b_scan_create(ctypes.byref(h), 0, 2, 4) == -2                  # no such mode
    assert L.nrsc5b_scan_create(ctypes.byref(h), 0, 0, 0) == -2                  # no channels
    assert L.nrsc5b_scan_create(None, 0, 0, 4) == -2
    assert L.nrsc5b_scan_push(None, None, 0) == -2
    assert L.nrsc5b_scan_result(None, None, None) == -2
    assert L.nrsc5b_chan_scan(None, None, None, 0) == -2


# ---------------------------------------------------------------- GPU tier

def _full_scale(rng, nch, nsamples):
    x = rng.integers(-32768, 32768, (nch, 2 * nsamples), dtype=np.int16)
    x[:, rng.integers(0, 2 * nsamples, 64)] = -32768
    return x


def _check_parity(res, raw, acc, want, mode, T):
    F, P, q, S, J, fs = so.geometry(mode)
    cw = so.windows(acc, mode)
    assert np.array_equal(raw[:, :6 * J].reshape(-1, 6, J), acc)
    assert np.array_equal(raw[:, 6 * J:12 * J].reshape(-1, 6, J), cw)
    for k, (g, w) in enumerate(zip(res, want)):
        assert g["timing"] == w["timing"] and g["detected"] == w["detected"], k
        for key in ("score", "threshold", "threshold_sideband", "score_lower", "score_upper", "symbols", "cfo_hz", "snr_db_lower", "snr_db_upper", "power_dbfs",
                    "power_dbfs_lower", "power_dbfs_upper"):
            a, b = g[key], w[key]
            assert (a == b) if math.isinf(b) else abs(a - b) <= 1e-9 * max(1.0, abs(b)), (k, key, a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,nch", [(FM, 1), (FM, 7), (FM, 119), (AM, 1), (AM, 7), (AM, 119)])
def test_kernel_equals_the_restatement_bit_for_bit(mode, nch):
    """Random full-scale cs16 plus a full-scale tone in channel 0's upper sideband, whose filter output saturates."""
    F, P, q, S, J, fs = so.geometry(mode)
    rng = np.random.default_rng(100 * mode + nch)
    T = 40 * S + 1234 if mode == FM else 300 * S + 77
    x = _full_scale(rng, nch, T)
    # a full-scale tone in the upper sideband of channel 0 for a while: its filter output saturates
    f_tone = 151e3 if mode == FM else 10400.0
    x[0, 2 * 5000:2 * 9000] = _iq(46000 * np.exp(2j * np.pi * f_tone / fs * np.arange(4000)))
    taps, kappa = scan.make_tables(BAND[mode])
    acc, want = so.scan(x, mode, taps, C[mode], kappa, C1[mode])
    zl, zu = so.sidebands(x[0], taps)
    assert np.abs(zu).max() >= 32767                                   # saturation is exercised
    with scan.Scanner(nch, BAND[mode]) as s:
        s.push(x)
        res, raw = s.result(raw=True)
    _check_parity(res, raw, acc, want, mode, T)
    pw = [int(r[12 * J]) & ((1 << 64) - 1) | (int(r[12 * J + 1]) << 64) for r in raw]
    assert pw == [int(np.sum(x[k].astype(np.int64) ** 2)) for k in range(nch)]


def _pieces(T, rng, mode):
    F, P, q, S, J, fs = so.geometry(mode)
    sizes = [0, 1, F // 3, 2 * S + 1, 0, q + 1, 7, 3 * F + 5, 1]
    cuts, pos = [0], 0
    for s in sizes:
        pos = min(T, pos + s)
        cuts.append(pos)
    while pos < T:
        pos = min(T, pos + int(rng.integers(1, 20 * S)))
        cuts.append(pos)
    return list(zip(cuts[:-1], cuts[1:]))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [FM, AM])
def test_pieces_of_every_size_equal_the_one_shot_scan(mode):
    import torch
    F, P, q, S, J, fs = so.geometry(mode)
    rng = np.random.default_rng(7 + mode)
    nch, T = 5, 60 * S + 999
    x = _full_scale(rng, nch, T)
    with scan.Scanner(nch, BAND[mode]) as s:
        s.push(x)
        one, raw1 = s.result(raw=True)
        s.reset()
        s.push(x[:, :2 * 3 * S])                                        # something to throw away
        s.reset()
        d = torch.from_numpy(x).cuda()
        for a, b in _pieces(T, rng, mode):
            part = d[:, 2 * a:2 * b].contiguous()
            s.push_device(part.data_ptr() if b > a else 0, max(2 * (b - a), 0), b - a)
            mid, _ = s.result(raw=True)                                 # a result between pushes changes nothing
        res, raw = s.result(raw=True)
    assert np.array_equal(raw, raw1)
    assert res == one


# ---- FM band: 23.814 MS/s, the 100 station slots (odd offsets -99..+99) of a 98.0 MHz-centred capture

WIDE = 23814000.0
FM_STATIONS = [  # (offset, psmi, scale x cu8 LSB, lead_in at 1 488 375 S/s, cfo_hz)
    (11, 1, 50.0, 1000, 0.0),            # strong, some 50 dB over the noise, with empty channels 100 - 400 kHz below it
    (13, 1, 0.5, 2200, 0.0),             # 40 dB below its neighbour
    (-23, 3, 4.0, 3100, 60.0),
    (41, 11, 2.0, 1700, -60.0),
]
CARRIER, ANALOG, SPUR_IN = -51, 67, -75


def _fm_band(seconds=0.62):
    import torch
    from nrsc5_b200 import synth
    dev = "cuda"
    n = int(seconds * 1488375)
    up = 16
    N = n * up
    t = torch.arange(N, dtype=torch.float64, device=dev)
    wide = torch.zeros(N, dtype=torch.complex128, device=dev)

    def place(z, m):
        ph = torch.remainder(t * (m * 100e3 / WIDE), 1.0) * (2 * math.pi)
        return z * torch.complex(torch.cos(ph), torch.sin(ph))

    for m, psmi, sc, lead, cfo in FM_STATIONS:
        cap = synth.make_fm(psmi=psmi, nframes=1, seed=40 + m, lead_in=lead, cfo_hz=cfo, tail_blocks=0)
        x = torch.from_numpy(cap.cu8[: 2 * n].astype(np.float64) - 127.0).to(dev).view(-1, 2)
        X = torch.fft.fft(torch.complex(x[:, 0].contiguous(), x[:, 1].contiguous()))
        Y = torch.zeros(N, dtype=torch.complex128, device=dev)
        Y[: n // 2] = X[: n // 2]
        Y[-(n - n // 2):] = X[n // 2:]
        wide += place(torch.fft.ifft(Y) * (up * sc), m)
        del X, Y
    wide += place(torch.full((N,), 2000.0, dtype=torch.complex128, device=dev), CARRIER)      # unmodulated carrier
    # analogue FM only: a 1 kHz tone at +-75 kHz deviation
    phi = 2 * math.pi * 75e3 / 1e3 * torch.sin(2 * math.pi * 1e3 * t / WIDE)
    wide += place(1500.0 * torch.complex(torch.cos(phi), torch.sin(phi)), ANALOG)
    wide += place(torch.full((N,), 3000.0, dtype=torch.complex128, device=dev) *
                  torch.exp(2j * math.pi * 160e3 / WIDE * t), SPUR_IN)                           # spur in the sideband
    g = torch.Generator(device=dev)
    g.manual_seed(3)
    iq = torch.stack([wide.real, wide.imag], -1) + torch.randn((N, 2), generator=g, device=dev, dtype=torch.float64) * 20.0
    del wide, t
    return torch.clamp(torch.round(iq), -32768, 32767).to(torch.int16).reshape(-1)


@pytest.fixture(scope="module")
def fm_band():
    import torch
    from nrsc5_b200 import channelizer as ch
    x = _fm_band()
    offs = list(range(-117, 118))                     # every 100 kHz grid point: a station's neighbours 100 - 400 kHz away
    nout = ch.outputs(x.numel())
    stride = (2 * nout + 64) & ~31
    d_out = torch.zeros((len(offs), stride), dtype=torch.int16, device="cuda")
    with ch.Channelizer(offs, input_cs16=True) as c:
        c.run_device(x.data_ptr(), x.numel(), d_out.data_ptr(), stride)
        torch.cuda.synchronize()
    with scan.Scanner(len(offs)) as s:
        s.push_device(d_out.data_ptr(), stride, nout)
        res = s.result()
    rows = scan.scan_band(x.cpu().numpy())           # the same through nrsc5b_chan_scan, default offsets
    assert [r["offset"] for r in rows] == offs
    assert [{k: v for k, v in r.items() if k != "offset"} for r in rows] == res
    return x, offs, d_out, nout, res


@pytest.mark.gpu
def test_fm_band_detects_exactly_the_hd_stations(fm_band):
    x, offs, d_out, nout, res = fm_band
    hd = {m for m, *_ in FM_STATIONS}
    got = {m for m, r in zip(offs, res) if r["detected"]}
    assert got == hd, [(m, round(r["score"], 4), round(r["threshold"], 4)) for m, r in zip(offs, res) if m in hd | got]
    S = 2160
    for m, psmi, sc, lead, cfo in FM_STATIONS:
        r = res[offs.index(m)]
        want = ((lead - 8) / 2) % S                   # the channeliser's group delay: 127.5 / 16 station samples
        assert min(abs(r["timing"] - want), S - abs(r["timing"] - want)) <= 4, (m, r["timing"], want)
        if cfo:
            assert abs(r["cfo_hz"] - cfo) < 2.0, (m, r["cfo_hz"])
    pw = {m: r["power_dbfs_upper"] for m, r in zip(offs, res)}
    assert pw[11] - pw[13] == pytest.approx(40.0, abs=1.5)


@pytest.mark.gpu
def test_fm_band_detected_channels_reach_sync(fm_band):
    import nrsc5_b200
    from nrsc5_b200 import engine as eng
    x, offs, d_out, nout, res = fm_band
    det = [k for k, r in enumerate(res) if r["detected"]]
    out = d_out[:, : 2 * nout].cpu().numpy()
    with nrsc5_b200.Engine(nstreams=len(det), input_capacity=4 * nout + 4096, log_capacity=4 << 20, input_cs16=True) as e:
        for i, k in enumerate(det):
            e.push_cs16(i, out[k])
        e.process()
        for i, k in enumerate(det):
            assert any(t == eng.REC_SYNC for t, _ in e.drain(i)), offs[k]


@pytest.mark.gpu
@pytest.mark.parametrize("decim,rate", [(16, None), (32, 10000000)])
def test_chan_scan_equals_channelise_then_scan(decim, rate):
    import torch
    from nrsc5_b200 import channelizer as ch
    fs = rate or decim * ch.FM_RATE
    lim = ch.resampler_tables(rate, decim, "fm")[2] if rate else 59
    offs = [-lim, -3, 0, 2, lim]
    n = int(0.3 * fs)
    rng = np.random.default_rng(decim)
    t = np.arange(n)
    z = 40 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    y = _fm_channel(seed=9)[: int(0.3 * 744187.5)]
    from scipy.signal import resample
    z += resample(y, n) * np.exp(2j * np.pi * 200e3 * t / fs) / 8
    x = _iq(z)
    with ch.Channelizer(offs, input_cs16=True, decim=decim, rate=rate) as c, scan.Scanner(len(offs)) as s:
        s.scan_capture(c, x[: 2 * 1001])                       # in two pieces, the first shorter than any filter
        s.scan_capture(c, x[2 * 1001:])
        got, graw = s.result(raw=True)
        c.reset()
        s.reset()
        out = c.push(x)
        s.push(out)
        want, wraw = s.result(raw=True)
    assert np.array_equal(graw, wraw)
    assert got == want
    assert got[offs.index(2)]["detected"] and sum(r["detected"] for r in got) == 1


# ---- sideband SNR

@pytest.mark.gpu
def test_fm_sideband_snr_against_the_truth():
    """One station, independent noise per sideband (each noise band-limited to its own sideband) at generated
    per-sideband SNRs; the truth runs the same taps on the signal and the noise apart."""
    taps, kappa = scan.make_tables("fm")
    fs, F = 744187.5, 2048
    sig = _fm_channel(seed=21, nframes=2, gain=64.0)[: int(3.0 * fs)]
    n = sig.size
    f = np.fft.fftfreq(n) * fs
    rng = np.random.default_rng(4)
    sideband = {"lower": (f <= -120e3) & (f >= -185e3), "upper": (f >= 120e3) & (f <= 185e3)}

    def band_noise(mask):
        w = np.fft.fft(rng.standard_normal(n) + 1j * rng.standard_normal(n)) * mask
        return np.fft.ifft(w)

    def zpow(z):
        zl, zu = so.sidebands(_iq(z), taps)
        return {"lower": float(np.mean(zl[64:].astype(np.float64) ** 2) * 2), "upper": float(np.mean(zu[64:].astype(np.float64) ** 2) * 2)}

    ps = zpow(sig)
    unit = {s: zpow(band_noise(sideband[s]) * 100.0)[s] for s in ("lower", "upper")}
    cases = [(0.0, 0.0), (6.0, 6.0), (12.0, 12.0), (3.0, 9.0), (10.0, 4.0)]
    ys, truth = [], []
    for lo_db, up_db in cases:
        zs = sig.copy()
        for s, db in (("lower", lo_db), ("upper", up_db)):
            zs += band_noise(sideband[s]) * 100.0 * math.sqrt(ps[s] / unit[s] / 10 ** (db / 10))
        ys.append(_iq(zs))
        truth.append((lo_db, up_db))
    with scan.Scanner(len(ys)) as s:
        s.push(np.stack(ys))
        res = s.result()
    for (lo_db, up_db), r in zip(truth, res):
        assert abs(r["snr_db_lower"] - lo_db) <= 1.5 and abs(r["snr_db_upper"] - up_db) <= 1.5, (lo_db, up_db, r)
        if abs(lo_db - up_db) >= 6:
            assert (r["snr_db_lower"] > r["snr_db_upper"]) == (lo_db > up_db)


@pytest.mark.gpu
def test_fm_station_at_minus_3_db_is_detected_in_half_a_second():
    fs = 744187.5
    sig = _fm_channel(seed=22, gain=64.0, lead_in=500)[: int(0.5 * fs)]
    taps, _ = scan.make_tables("fm")
    zl, zu = so.sidebands(_iq(sig), taps)
    ps = float(np.mean(zu[64:].astype(np.float64) ** 2) * 2)
    rng = np.random.default_rng(8)
    # white noise of the same per-sideband power through the taps (the taps' noise gain is sum |g|^2 / 2^30)
    g2 = float(np.sum(taps.astype(np.float64) ** 2)) / 2 ** 30
    sigma = math.sqrt(ps / 10 ** (-3 / 10) / g2 / 2)
    y = _iq(sig + sigma * (rng.standard_normal(sig.size) + 1j * rng.standard_normal(sig.size)))
    with scan.Scanner(1) as s:
        s.push(y[None])
        r = s.result()[0]
    assert r["detected"], r


# ---- AM band

AM_STATIONS = [  # (offset, psmi 1 = MA1 with carrier / 2 = MA3, gain, lead_in, cfo_hz)
    (-40, 1, 1.0, 900, 0.0),
    (-7, 2, 1.0, 1500, 25.0),
    (12, 1, 0.3, 700, -25.0),
    (33, 2, 0.5, 2100, 0.0),
]


def _am_band(seed=5, noise_lsb=60.0):
    """The AM_STATIONS in one cs16 capture at 1 488 375 S/s: each interpolated by 32 in the frequency domain (no images
    at multiples of 46.5 kHz, which a polyphase interpolator leaves some 40 dB down and which are CP-periodic signals
    of their own), moved to its offset, with a white noise floor some 60 dB under the stations' carriers (a lower one
    lets the scan hear the channeliser's -87 dB aliases, which are CP-periodic too)."""
    from nrsc5_b200 import synth_am
    caps = [synth_am.make_am_ma1(nframes=2, seed=60 + m, lead_in=lead, psmi=psmi, cfo_hz=cfo, noise_lsb=0.0).cs16
            for m, psmi, gain, lead, cfo in AM_STATIONS]
    n = min(c.size for c in caps) // 2
    N = 32 * n
    t = np.arange(N, dtype=np.float64)
    wide = np.zeros(N, dtype=np.complex128)
    for c, (m, psmi, gain, lead, cfo) in zip(caps, AM_STATIONS):
        X = np.fft.fft(c[0:2 * n:2] + 1j * c[1:2 * n:2].astype(np.float64))
        Y = np.zeros(N, dtype=np.complex128)
        Y[: n // 2] = X[: n // 2]
        Y[-(n - n // 2):] = X[n // 2:]
        wide += np.fft.ifft(Y) * (32 * gain) * np.exp(2j * np.pi * ((80 * m) % 11907) / 11907.0 * t)
    rng = np.random.default_rng(seed)
    wide += noise_lsb * (rng.standard_normal(N) + 1j * rng.standard_normal(N))
    return _iq(wide)


@pytest.mark.gpu
def test_am_band():
    from nrsc5_b200 import channelizer as ch
    x = _am_band()
    offs = list(range(-59, 59))
    with ch.Channelizer(offs, input_cs16=True, band="am") as c, scan.Scanner(len(offs), "am") as s:
        s.scan_capture(c, x)
        res = s.result()
    got = {m for m, r in zip(offs, res) if r["detected"]}
    hd = {m for m, *_ in AM_STATIONS}
    assert got == hd, [(m, r["score"], r["score_lower"], r["score_upper"]) for m, r in zip(offs, res) if r["detected"]]
    for m, psmi, gain, lead, cfo in AM_STATIONS:
        r = res[offs.index(m)]
        want = (lead - 8) % 270                       # the channeliser's group delay: 255.5 / 32 station samples
        assert min(abs(r["timing"] - want), 270 - abs(r["timing"] - want)) <= 2, (m, r["timing"], want)
        if cfo:
            assert abs(r["cfo_hz"] - cfo) < 2.0, (m, r["cfo_hz"])


# ---- false alarms

@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(5))
def test_no_false_alarm_on_noise(seed):
    import torch
    for mode, nch, secs in ((FM, 119, 1.0), (AM, 118, 2.0)):
        fs = so.geometry(mode)[5]
        n = int(secs * fs)
        g = torch.Generator(device="cuda")
        g.manual_seed(1000 * seed + mode)
        x = torch.clamp(torch.round(torch.randn((nch, 2 * n), generator=g, device="cuda") * 800.0), -32768, 32767).to(torch.int16)
        with scan.Scanner(nch, BAND[mode]) as s:
            s.push_device(x.data_ptr(), 2 * n, n)
            res = s.result()
        assert not any(r["detected"] for r in res), [(k, r["score"], r["threshold"]) for k, r in enumerate(res) if r["detected"]]
        assert all(r["symbols"] >= 32 for r in res)
