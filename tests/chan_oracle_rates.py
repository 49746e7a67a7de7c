"""TEST INFRASTRUCTURE ONLY.  The channeliser's FM plans at D x 744 187.5 S/s, D = 32, 16 or 8 (include/nrsc5_b200.h:
nrsc5b_chan_create_fm), restated in numpy, one-shot and streamed, for cu8 and cs16 input: exact integer arithmetic on
the tables the library publishes.  Output n's window starts at input sample D n; the tap scale is 2^14 D, so the
rounding shifts are s = 13 - log2(32 / D) (cu8) and t = 19 - log2(32 / D) (cs16).  With D = 32 it is
oracle/chan_oracle.py and tests/chan_oracle_cs16.py."""
import numpy as np

PERIOD, TAPS, MIX = 11907, 256, 1600
BLOCK = 4096                                                                       # outputs gathered at a time


def shifts(decim: int):
    """(s, t): the cu8 and cs16 rounding shifts of the plan."""
    lq = {32: 0, 16: 1, 8: 2}[decim]
    return 13 - lq, 19 - lq


def outputs_of(samples: int, decim: int) -> int:
    """N_D(T): outputs whose 256-sample windows lie within the first T complex samples."""
    return (samples - TAPS) // decim + 1 if samples >= TAPS else 0


def channelize(x: np.ndarray, offsets, taps: np.ndarray, phasor: np.ndarray, decim: int, n0: int = 0) -> np.ndarray:
    """x: uint8 (cu8) or int16 (cs16), I/Q interleaved, whole complex samples -> int16 [nch][2 * nout].  n0: index of
    the first output when x is a slice of a longer capture starting at its sample D * n0 (the mixer runs on)."""
    a = np.asarray(x).reshape(-1)
    assert a.dtype in (np.uint8, np.int16) and a.size % 2 == 0
    assert taps.shape[1] == TAPS
    cu8 = a.dtype == np.uint8
    s, t = shifts(decim)
    nout = outputs_of(a.size // 2, decim)
    xr = a[0::2].astype(np.int64) - (127 if cu8 else 0)
    xi = a[1::2].astype(np.int64) - (127 if cu8 else 0)
    out = np.zeros((len(offsets), 2 * max(nout, 0)), dtype=np.int16)
    # float64 holds these sums exactly (products below 2^30, 256 of them below 2^38 < 2^53)
    wr = taps[:, :, 0].astype(np.float64).T                                        # [256][nch]
    wi = taps[:, :, 1].astype(np.float64).T
    step = np.array([(MIX * int(m)) % PERIOD for m in offsets], dtype=np.int64)
    for b0 in range(0, nout, BLOCK):
        nb = min(BLOCK, nout - b0)
        idx = np.arange(b0, b0 + nb)[:, None] * decim + np.arange(TAPS)[None, :]
        XR, XI = xr[idx].astype(np.float64), xi[idx].astype(np.float64)
        ar = (XR @ wr - XI @ wi).astype(np.int64)
        ai = (XI @ wr + XR @ wi).astype(np.int64)
        if cu8:
            vr, vi = (ar + (1 << (s - 1))) >> s, (ai + (1 << (s - 1))) >> s
        else:
            vr = np.clip((ar + (1 << (t - 1))) >> t, -32768, 32767)
            vi = np.clip((ai + (1 << (t - 1))) >> t, -32768, 32767)
        n = np.arange(b0, b0 + nb, dtype=np.int64) + int(n0)
        q = (step[None, :] * (n % PERIOD)[:, None]) % PERIOD                       # [nb][nch]
        pr = phasor[q, 0].astype(np.int64)
        pi = phasor[q, 1].astype(np.int64)
        zr = (vr * pr + vi * pi + (1 << 14)) >> 15                                # v * conj(P)
        zi = (vi * pr - vr * pi + (1 << 14)) >> 15
        out[:, 2 * b0: 2 * (b0 + nb): 2] = np.clip(zr, -32768, 32767).astype(np.int16).T
        out[:, 2 * b0 + 1: 2 * (b0 + nb): 2] = np.clip(zi, -32768, 32767).astype(np.int16).T
    return out


def channelize_stream(chunks, offsets, taps: np.ndarray, phasor: np.ndarray, decim: int):
    """The streaming form (nrsc5b_chan_push*): a push taking T to T' emits outputs N(T) .. N(T') - 1, computed from
    carry + chunk with the mixer at the absolute index N(T), and keeps the samples from D N(T') on (at most 255).
    Returns one int16 [nch][2 * n] array per push."""
    carry, pushed, outs = None, 0, []
    for chunk in chunks:
        c = np.asarray(chunk).reshape(-1)
        assert c.size % 2 == 0, "pushes are whole complex samples"
        first, last = outputs_of(pushed, decim), outputs_of(pushed + c.size // 2, decim)
        held = c if carry is None else np.concatenate([carry, c])                 # starts at sample D N(T)
        n = last - first
        outs.append(channelize(held[: 2 * (decim * n + TAPS - decim)] if n > 0 else held[:0], offsets, taps, phasor, decim, n0=first))
        pushed += c.size // 2
        carry = held[2 * decim * n:]
        assert carry.size == 2 * (pushed - decim * last) <= 2 * (TAPS - 1)
    return outs
